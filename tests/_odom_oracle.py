"""ctypes access to the odometry-model oracle (tests/host/pf_odom_oracle.c, which includes tests/host/pf_beam_oracle.c and through it
the likelihood-field, recovery and PF oracles unchanged).  Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

import _assoc_oracle
import _beam_oracle as BM
import _lfield_oracle as LF
import _oracle
import _recovery_oracle as R
from _oracle import f64

SRC = os.path.join(_oracle.ROOT, "tests", "host", "pf_odom_oracle.c")
_LIBS = {}
ALPHA_DEFAULT = (0.2, 0.2, 0.2, 0.2)


def load(libm=False):
    """the oracle library (contract math, or glibc libm with libm=True), built here on first use"""
    if libm not in _LIBS:
        out = os.path.join(_oracle.ROOT, "tests", "host", "libpf_odom_oracle%s.so" % ("_libm" if libm else ""))
        deps = [SRC, BM.SRC, LF.SRC, R.SRC] + [os.path.join(_oracle.ROOT, d) for d in (
            "oracle/pf_oracle.c", "oracle/oracle.h", "include/pf_contract_math.h", "include/pf_odom_math.h", "include/fs_ekf_math.h")]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            subprocess.run(["/usr/bin/gcc"] + _assoc_oracle.CFLAGS + (["-DPF_ORACLE_LIBM"] if libm else []) + ["-shared", "-o", out, SRC, "-lm"],
                           check=True)
        _LIBS[libm] = _declare(C.CDLL(out))
    return _LIBS[libm]


def _declare(L):
    """the beam oracle's declarations (the same symbols are in this library) and the odometry entry points"""
    vp, dp, u8p, sz, d = C.c_void_p, _oracle.c_dp, C.POINTER(C.c_uint8), C.c_size_t, C.c_double
    L.orc_bm_new.argtypes, L.orc_bm_new.restype = [C.POINTER(_oracle.PfConfig), C.c_uint64], vp
    L.orc_bm_lf.argtypes, L.orc_bm_lf.restype = [vp], vp
    L.orc_lf_rec.argtypes, L.orc_lf_rec.restype = [vp], vp
    L.orc_rec_pf.argtypes, L.orc_rec_pf.restype = [vp], vp
    L.orc_bm_beams.restype = L.orc_bm_weights.restype = L.orc_lf_beams.restype = L.orc_lf_weights.restype = C.c_long
    L.orc_pf_count.restype = L.orc_pf_last_indices.restype = C.c_size_t
    for name in ("orc_bm_free", "orc_bm_clear", "orc_lf_clear", "orc_rec_state", "orc_rec_upload"):
        getattr(L, name).restype = None
    for name, args in (("orc_bm_free", [vp]), ("orc_bm_clear", [vp]), ("orc_bm_set", [vp, u8p, sz, sz, dp]),
                       ("orc_bm_update_beam", [vp, dp, sz, d, d]), ("orc_lf_clear", [vp]), ("orc_lf_set", [vp, u8p, sz, sz, dp]),
                       ("orc_lf_update_scan", [vp, dp, sz, d, d]),
                       ("orc_rec_enable", [vp, d, d, dp]), ("orc_rec_state", [vp, dp, C.POINTER(C.c_uint64)]),
                       ("orc_rec_init_region_with_uniforms", [vp, dp, dp]), ("orc_rec_init_state", [vp, dp]),
                       ("orc_rec_upload", [vp, dp, sz]), ("orc_rec_predict_with_draws", [vp, dp, dp, dp, dp]),
                       ("orc_rec_update", [vp, dp, sz]), ("orc_rec_resample_with_uniforms", [vp, dp, sz]),
                       ("orc_pf_count", [vp]), ("orc_pf_get_particles", [vp, dp]), ("orc_pf_estimate", [vp, dp, dp]),
                       ("orc_pf_last_indices", [vp, _oracle.c_u32p, sz]), ("orc_pf_set_fast_search", [vp, C.c_int]),
                       ("orc_pf_set_threads", [vp, C.c_int]),
                       ("orc_od_increment", [dp, dp, dp]), ("orc_od_alpha_ok", [dp]), ("orc_od_predict", [vp, dp, dp, dp, dp])):
        getattr(L, name).argtypes = args
    return L


def _dp(a):
    return None if a is None else a.ctypes.data_as(_oracle.c_dp)


def increment(odom_prev, odom_cur, alpha=ALPHA_DEFAULT, libm=False):
    """(rot1, trans, rot2, s_rot1, s_trans, s_rot2) of one call, or None when refused"""
    o, a, out = f64(list(odom_prev) + list(odom_cur)), f64(alpha), np.empty(6)
    return None if load(libm).orc_od_increment(_dp(o), _dp(a), _dp(out)) != 0 else out


class OracleOdom(BM.OracleBeam):
    """OracleBeam with the odometry motion model: set_odom_noise / predict_odom / step_odom / step_scan_odom / step_beam_odom.  The
    velocity-model methods stay, so one oracle mirrors a handle that mixes the two motion models."""

    def __init__(self, n, threshold=0.5, range_noise=0.2, velocity_noise=2.0, yaw_rate_noise=np.deg2rad(40.0), dt=0.1, seed=42, mode=0,
                 max_particles=None, kld_epsilon=0.05, kld_z=2.326, libm=False, fast_search=True, threads=1):
        self.L = load(libm)
        self.cfg = _oracle.PfConfig(n, threshold, range_noise, velocity_noise, yaw_rate_noise, dt, mode, 0,
                                    max_particles if max_particles is not None else n, kld_epsilon, kld_z)
        self.bm = self.L.orc_bm_new(C.byref(self.cfg), seed)
        if not self.bm:
            raise ValueError("InvalidParameter")
        self.lf = self.L.orc_bm_lf(self.bm)
        self.r = self.L.orc_lf_rec(self.lf)
        self.h = self.L.orc_rec_pf(self.r)
        self.cap = int(self.cfg.max_particles)
        self.alpha = f64(ALPHA_DEFAULT)
        self.L.orc_pf_set_fast_search(self.h, int(fast_search))
        self.L.orc_pf_set_threads(self.h, int(threads))

    def set_odom_noise(self, alpha):
        a = f64(alpha)
        if a.size != 4 or not self.L.orc_od_alpha_ok(_dp(a)):
            return -1
        self.alpha = a
        return 0

    def predict_odom(self, odom_prev, odom_cur, z3=None, inj4=None):
        o = f64(list(odom_prev) + list(odom_cur))
        z, i4 = (None if v is None else f64(v) for v in (z3, inj4))
        return self.L.orc_od_predict(self.r, _dp(o), _dp(self.alpha), _dp(z), _dp(i4))

    def step_odom(self, odom_prev, odom_cur, obs):
        """try_step with odometry: predict_odom, update, resample -> (estimate, resampled)"""
        assert self.predict_odom(odom_prev, odom_cur) == 0 and self.update(obs) == 0
        did = self.resample()
        return self.estimate(), did

    def step_scan_odom(self, odom_prev, odom_cur, ranges, angle_min, angle_inc):
        assert self.predict_odom(odom_prev, odom_cur) == 0 and self.update_scan(ranges, angle_min, angle_inc) == 0
        did = self.resample()
        return self.estimate(), did

    def step_beam_odom(self, odom_prev, odom_cur, ranges, angle_min, angle_inc):
        assert self.predict_odom(odom_prev, odom_cur) == 0 and self.update_beam(ranges, angle_min, angle_inc) == 0
        did = self.resample()
        return self.estimate(), did
