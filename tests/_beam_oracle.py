"""ctypes access to the beam-model oracle (tests/host/pf_beam_oracle.c, which includes tests/host/pf_lfield_oracle.c and through it
the recovery and PF oracles unchanged).  Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

import _assoc_oracle
import _lfield_oracle as LF
import _oracle
import _recovery_oracle as R
from _oracle import f64

SRC = os.path.join(_oracle.ROOT, "tests", "host", "pf_beam_oracle.c")
_LIBS = {}


def load(libm=False):
    """the oracle library (contract math, or glibc libm with libm=True), built here on first use"""
    if libm not in _LIBS:
        out = os.path.join(_oracle.ROOT, "tests", "host", "libpf_beam_oracle%s.so" % ("_libm" if libm else ""))
        deps = [SRC, LF.SRC, R.SRC] + [os.path.join(_oracle.ROOT, d) for d in ("oracle/pf_oracle.c", "oracle/oracle.h",
                                                                              "include/pf_contract_math.h")]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            subprocess.run(["/usr/bin/gcc"] + _assoc_oracle.CFLAGS + (["-DPF_ORACLE_LIBM"] if libm else []) + ["-shared", "-o", out, SRC, "-lm"],
                           check=True)
        L = C.CDLL(out)
        vp, dp, u8p, sz, d = C.c_void_p, _oracle.c_dp, C.POINTER(C.c_uint8), C.c_size_t, C.c_double
        L.orc_bm_new.argtypes, L.orc_bm_new.restype = [C.POINTER(_oracle.PfConfig), C.c_uint64], vp
        L.orc_bm_lf.argtypes, L.orc_bm_lf.restype = [vp], vp
        L.orc_lf_rec.argtypes, L.orc_lf_rec.restype = [vp], vp
        L.orc_rec_pf.argtypes, L.orc_rec_pf.restype = [vp], vp
        L.orc_bm_cast.argtypes, L.orc_bm_cast.restype = [vp, d, d, d], d
        L.orc_bm_beams.restype = L.orc_bm_weights.restype = L.orc_lf_beams.restype = L.orc_lf_weights.restype = C.c_long
        L.orc_pf_count.restype = L.orc_pf_last_indices.restype = C.c_size_t
        for name in ("orc_bm_free", "orc_bm_clear", "orc_bm_info", "orc_bm_clearance", "orc_bm_chessboard", "orc_bm_raycast",
                     "orc_lf_clear", "orc_lf_info", "orc_lf_tables", "orc_rec_state", "orc_rec_upload"):
            getattr(L, name).restype = None
        for name, args in (("orc_bm_free", [vp]), ("orc_bm_clear", [vp]), ("orc_bm_set", [vp, u8p, sz, sz, dp]),
                           ("orc_bm_info", [vp, C.POINTER(C.c_uint64)]), ("orc_bm_clearance", [vp, u8p]),
                           ("orc_bm_chessboard", [u8p, sz, sz, u8p]), ("orc_bm_raycast", [vp, dp, sz, sz, d, d, dp]),
                           ("orc_bm_beams", [vp, dp, sz, d, d, dp]), ("orc_bm_weights", [vp, dp, sz, dp, sz, d, d, dp]),
                           ("orc_bm_update_beam", [vp, dp, sz, d, d]),
                           ("orc_lf_clear", [vp]), ("orc_lf_set", [vp, u8p, sz, sz, dp]), ("orc_lf_info", [vp, C.POINTER(C.c_uint64)]),
                           ("orc_lf_tables", [vp, dp, dp]), ("orc_lf_beams", [vp, dp, sz, d, d, dp]),
                           ("orc_lf_weights", [vp, dp, sz, dp, sz, d, d, dp]), ("orc_lf_update_scan", [vp, dp, sz, d, d]),
                           ("orc_rec_enable", [vp, d, d, dp]), ("orc_rec_state", [vp, dp, C.POINTER(C.c_uint64)]),
                           ("orc_rec_init_region_with_uniforms", [vp, dp, dp]), ("orc_rec_init_state", [vp, dp]),
                           ("orc_rec_upload", [vp, dp, sz]), ("orc_rec_predict_with_draws", [vp, dp, dp, dp, dp]),
                           ("orc_rec_update", [vp, dp, sz]), ("orc_rec_resample_with_uniforms", [vp, dp, sz]),
                           ("orc_pf_count", [vp]), ("orc_pf_get_particles", [vp, dp]), ("orc_pf_estimate", [vp, dp, dp]),
                           ("orc_pf_last_indices", [vp, _oracle.c_u32p, sz]), ("orc_pf_set_fast_search", [vp, C.c_int]),
                           ("orc_pf_set_threads", [vp, C.c_int])):
            getattr(L, name).argtypes = args
        _LIBS[libm] = L
    return _LIBS[libm]


def _dp(a):
    return None if a is None else a.ctypes.data_as(_oracle.c_dp)


def _u8(mask):
    return np.ascontiguousarray(np.asarray(mask) != 0, dtype=np.uint8)


def chessboard(mask, libm=False):
    """the oracle's clearance table of a mask: (W, H) uint8"""
    m = _u8(mask)
    out = np.empty(m.shape, dtype=np.uint8)
    load(libm).orc_bm_chessboard(m.ctypes.data_as(C.POINTER(C.c_uint8)), m.shape[0], m.shape[1], out.ctypes.data_as(C.POINTER(C.c_uint8)))
    return out


BEAM_DEFAULTS = dict(sigma_hit=0.2, z_hit=0.95, z_short=0.1, z_max=0.05, z_rand=0.05, lambda_short=0.1, max_range=30.0, max_beams=60)


class OracleBeam(LF.OracleLField):
    """OracleLField with a beam map as well: set_beam_map / update_beam / step_beam / beam_weights / raycast (the engine's keyword
    arguments); the likelihood-field methods stay, so one oracle mirrors a handle that mixes the models"""

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
        self.L.orc_pf_set_fast_search(self.h, int(fast_search))
        self.L.orc_pf_set_threads(self.h, int(threads))

    def __del__(self):
        if getattr(self, "bm", None):
            self.L.orc_bm_free(self.bm)
            self.bm = self.lf = self.r = None

    def set_beam_map(self, obstacles, resolution, **kw):
        c = dict(BEAM_DEFAULTS)
        c.update(kw)
        m = _u8(obstacles)
        cfg = f64([resolution, c["sigma_hit"], c["z_hit"], c["z_short"], c["z_max"], c["z_rand"], c["lambda_short"], c["max_range"],
                   c["max_beams"]])
        return self.L.orc_bm_set(self.bm, m.ctypes.data_as(C.POINTER(C.c_uint8)), m.shape[0], m.shape[1], _dp(cfg))

    def clear_beam_map(self):
        self.L.orc_bm_clear(self.bm)

    def beam_info(self):
        """(W, H, L)"""
        out = (C.c_uint64 * 3)()
        self.L.orc_bm_info(self.bm, out)
        return tuple(int(v) for v in out)

    def clearance(self):
        W, H, _ = self.beam_info()
        out = np.empty((W, H), dtype=np.uint8)
        self.L.orc_bm_clearance(self.bm, out.ctypes.data_as(C.POINTER(C.c_uint8)))
        return out

    def raycast(self, poses, n_beams, angle_min, angle_inc):
        """expected ranges (n, n_beams) of poses (n, 3)"""
        p = f64(poses).reshape(-1, 3)
        out = np.empty((p.shape[0], int(n_beams)))
        self.L.orc_bm_raycast(self.bm, _dp(p), p.shape[0], int(n_beams), float(angle_min), float(angle_inc), _dp(out))
        return out

    def beam_beams(self, ranges, angle_min, angle_inc):
        """the used beams (k, 2) = (r_i, a_i), or None when refused"""
        r = f64(ranges).ravel()
        out = np.empty((max(r.size, 1), 2))
        k = self.L.orc_bm_beams(self.bm, _dp(r), r.size, float(angle_min), float(angle_inc), _dp(out))
        return None if k < 0 else out[:k].copy()

    def beam_weights(self, pose3, ranges, angle_min, angle_inc):
        """raw weights of poses (n, 3) under one scan (None when refused), without touching the filter"""
        p, r = f64(pose3).reshape(-1, 3), f64(ranges).ravel()
        w = np.empty(p.shape[0])
        k = self.L.orc_bm_weights(self.bm, _dp(p), p.shape[0], _dp(r), r.size, float(angle_min), float(angle_inc), _dp(w))
        return None if k < 0 else w

    def update_beam(self, ranges, angle_min, angle_inc):
        r = f64(ranges).ravel()
        return self.L.orc_bm_update_beam(self.bm, _dp(r), r.size, float(angle_min), float(angle_inc))

    def step_beam(self, u, ranges, angle_min, angle_inc):
        """try_step with a scan under the beam model: predict, update_beam, resample -> (estimate, resampled)"""
        assert self.predict(u) == 0 and self.update_beam(ranges, angle_min, angle_inc) == 0
        did = self.resample()
        return self.estimate(), did
