"""ctypes access to the occupancy grid mapping oracle (tests/host/ogm_oracle.c).  Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

import _assoc_oracle
import _oracle

SRC = os.path.join(_oracle.ROOT, "tests", "host", "ogm_oracle.c")
_LIBS = {}
DEFAULTS = dict(resolution=0.5, width=100, height=100, prior_log_odds=0.0, occupied_log_odds=0.85, free_log_odds=-0.4,
                max_log_odds=5.0, min_log_odds=-5.0)


def load(libm=False):
    """the oracle library (contract math, or glibc libm with libm=True), built here on first use"""
    if libm not in _LIBS:
        out = os.path.join(_oracle.ROOT, "tests", "host", "libogm_oracle%s.so" % ("_libm" if libm else ""))
        deps = [SRC, os.path.join(_oracle.ROOT, "include", "pf_contract_math.h")]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            subprocess.run(["/usr/bin/gcc"] + _assoc_oracle.CFLAGS + (["-DPF_ORACLE_LIBM"] if libm else []) + ["-shared", "-o", out, SRC, "-lm"],
                           check=True)
        L = C.CDLL(out)
        dp, sz, d = _oracle.c_dp, C.c_size_t, C.c_double
        for name in ("orc_ogm_update_scan", "orc_ogm_update_scans", "orc_ogm_census", "orc_ogm_obstacles"):
            getattr(L, name).restype = None
        L.orc_ogm_update_scan.argtypes = [dp, dp, sz, sz, d, d, d, dp, sz, d, d]
        L.orc_ogm_update_scans.argtypes = [dp, dp, sz, sz, dp, sz, dp, sz, d, d]
        L.orc_ogm_census.argtypes = [dp, sz, sz, dp, sz, dp, sz, d, d, C.POINTER(C.c_uint64)]
        L.orc_ogm_obstacles.argtypes = [dp, sz, d, C.POINTER(C.c_uint8)]
        L.orc_ogm_line.argtypes, L.orc_ogm_line.restype = [C.c_int32] * 4 + [C.POINTER(C.c_int32), sz], sz
        L.orc_ogm_is_libm.restype = C.c_int
        _LIBS[libm] = L
    return _LIBS[libm]


def _dp(a):
    return a.ctypes.data_as(_oracle.c_dp)


def _cfg(cfg):
    return np.array([cfg["resolution"], cfg["prior_log_odds"], cfg["occupied_log_odds"], cfg["free_log_odds"], cfg["max_log_odds"],
                     cfg["min_log_odds"]], dtype=np.float64)


def _batch(poses, ranges):
    p = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(-1, 3))
    r = np.ascontiguousarray(np.asarray(ranges, dtype=np.float64).reshape(p.shape[0], -1) if p.shape[0] else np.zeros((0, 0)))
    return p, r


class OracleOgm:
    """OccupancyGridMap on the CPU: grid (W, H) f64 log-odds, the keyword config of OccupancyGridConfig"""

    def __init__(self, libm=False, **cfg):
        self.cfg = dict(DEFAULTS, **cfg)
        self.L = load(libm)
        self.W, self.H = int(self.cfg["width"]), int(self.cfg["height"])
        self.grid = np.full((self.W, self.H), float(self.cfg["prior_log_odds"]))
        self._c = _cfg(self.cfg)

    def update_with_scan(self, x, y, yaw, ranges, angle_min, angle_inc):
        r = np.ascontiguousarray(np.asarray(ranges, dtype=np.float64).ravel())
        self.L.orc_ogm_update_scan(_dp(self.grid), _dp(self._c), self.W, self.H, float(x), float(y), float(yaw), _dp(r), r.size,
                                   float(angle_min), float(angle_inc))

    def update_with_scans(self, poses, ranges, angle_min, angle_inc):
        p, r = _batch(poses, ranges)
        self.L.orc_ogm_update_scans(_dp(self.grid), _dp(self._c), self.W, self.H, _dp(p), p.shape[0], _dp(r), r.shape[1] if r.ndim == 2 else 0,
                                    float(angle_min), float(angle_inc))

    def census(self, poses, ranges, angle_min, angle_inc):
        """(events, most updates of one cell, beams with a repeated cell, longest ray) of a batch on this map's shape"""
        p, r = _batch(poses, ranges)
        out = (C.c_uint64 * 4)()
        self.L.orc_ogm_census(_dp(self._c), self.W, self.H, _dp(p), p.shape[0], _dp(r), r.shape[1] if r.ndim == 2 else 0, float(angle_min),
                              float(angle_inc), out)
        return tuple(int(v) for v in out)

    def obstacles(self, threshold=0.5):
        g = np.ascontiguousarray(self.grid)
        m = np.empty(g.shape, dtype=np.uint8)
        self.L.orc_ogm_obstacles(_dp(g), g.size, float(threshold), m.ctypes.data_as(C.POINTER(C.c_uint8)))
        return m


def line(x0, y0, x1, y1, libm=False):
    """bresenham_line's cells as an (n, 2) int array"""
    n = max(abs(x1 - x0), abs(y1 - y0)) * 2 + 2
    out = np.empty((n, 2), dtype=np.int32)
    k = load(libm).orc_ogm_line(x0, y0, x1, y1, out.ctypes.data_as(C.POINTER(C.c_int32)), n)
    return out[:k]
