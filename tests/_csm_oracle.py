"""ctypes access to the correlative scan matching oracle (tests/host/csm_oracle.c).  Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

import _assoc_oracle
import _oracle

SRC = os.path.join(_oracle.ROOT, "tests", "host", "csm_oracle.c")
_LIBS = {}
# CorrelativeScanMatcherConfig::default()
DEFAULTS = dict(linear_search_range=1.0, angular_search_range=0.2, linear_step=0.1, angular_step=0.02, grid_resolution=0.05)
FIELDS = ("linear_search_range", "angular_search_range", "linear_step", "angular_step", "grid_resolution")


def load(libm=False):
    """the oracle library (contract math, or glibc libm with libm=True), built here on first use"""
    if libm not in _LIBS:
        out = os.path.join(_oracle.ROOT, "tests", "host", "libcsm_oracle%s.so" % ("_libm" if libm else ""))
        deps = [SRC, os.path.join(_oracle.ROOT, "include", "pf_contract_math.h")]
        if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
            subprocess.run(["/usr/bin/gcc"] + _assoc_oracle.CFLAGS + (["-DPF_ORACLE_LIBM"] if libm else []) + ["-shared", "-o", out, SRC, "-lm"],
                           check=True)
        L = C.CDLL(out)
        dp, sz = _oracle.c_dp, C.c_size_t
        L.orc_csm_match.restype = None
        L.orc_csm_match.argtypes = [dp, dp, sz, dp, dp, sz, dp, dp, dp, C.POINTER(C.c_uint64)]
        L.orc_csm_table.restype = sz
        L.orc_csm_table.argtypes = [dp, dp, sz, C.c_double, C.POINTER(C.c_int32), dp, sz, C.POINTER(C.c_int32)]
        L.orc_csm_score.restype = C.c_double
        L.orc_csm_score.argtypes = [dp, dp, sz, dp, dp, sz, dp, C.c_double]
        L.orc_csm_is_libm.restype = C.c_int
        _LIBS[libm] = L
    return _LIBS[libm]


def _a(v):
    return np.ascontiguousarray(np.asarray(v, dtype=np.float64).ravel())


def _dp(a):
    return a.ctypes.data_as(_oracle.c_dp)


def cfg_array(cfg=None):
    c = dict(DEFAULTS, **(cfg or {}))
    return np.array([float(c[k]) for k in FIELDS])


def match(rx, ry, qx, qy, pose, cfg=None, libm=False):
    """correlative_scan_match: (x, y, yaw, score, converged, candidates)"""
    rx, ry, qx, qy, p, c = _a(rx), _a(ry), _a(qx), _a(qy), _a(pose), cfg_array(cfg)
    assert rx.size == ry.size and qx.size == qy.size and p.size == 3
    out = np.zeros(5)
    n = C.c_uint64()
    load(libm).orc_csm_match(_dp(rx), _dp(ry), rx.size, _dp(qx), _dp(qy), qx.size, _dp(p), _dp(c), _dp(out), C.byref(n))
    return float(out[0]), float(out[1]), float(out[2]), float(out[3]), bool(out[4]), int(n.value)


def table(rx, ry, res, libm=False):
    """the lookup table as ({(ix, iy): weight}, R)"""
    rx, ry = _a(rx), _a(ry)
    L = load(libm)
    R = C.c_int32()
    n = L.orc_csm_table(_dp(rx), _dp(ry), rx.size, float(res), None, None, 0, C.byref(R))
    keys = np.empty((max(n, 1), 2), dtype=np.int32)
    vals = np.empty(max(n, 1))
    L.orc_csm_table(_dp(rx), _dp(ry), rx.size, float(res), keys.ctypes.data_as(C.POINTER(C.c_int32)), _dp(vals), n, C.byref(R))
    return {(int(k[0]), int(k[1])): float(v) for k, v in zip(keys[:n], vals[:n])}, int(R.value)


def score(rx, ry, qx, qy, pose, res, libm=False):
    rx, ry, qx, qy, p = _a(rx), _a(ry), _a(qx), _a(qy), _a(pose)
    return float(load(libm).orc_csm_score(_dp(rx), _dp(ry), rx.size, _dp(qx), _dp(qy), qx.size, _dp(p), float(res)))


def grid_points(obstacles, res):
    """the cell centres of a (W, H) obstacle mask in cell order: (((ix + 0.5) - W / 2.0) * res, ((iy + 0.5) - H / 2.0) * res)"""
    W, H = obstacles.shape
    ix, iy = np.nonzero(obstacles)
    return ((ix.astype(np.float64) + 0.5) - W / 2.0) * res, ((iy.astype(np.float64) + 0.5) - H / 2.0) * res


def scan_points(ranges, angle_min, angle_inc):
    """the finite beams of a scan as points in the robot frame: r cos(angle_min + i inc), r sin(...)"""
    r = np.asarray(ranges, dtype=np.float64)
    a = angle_min + np.arange(r.size) * angle_inc
    ok = np.isfinite(r) & (r > 0.0)
    return r[ok] * np.cos(a[ok]), r[ok] * np.sin(a[ok])


# the scan-matched mapping loop (test_csm_oracle.py, test_gpu_csm.py, the README): +-0.25 m / +-0.06 rad windows at 2.5 cm /
# 0.005 rad steps (21 x 21 x 25 candidates) on the scenario's 5 cm grid
MAP_CFG = dict(linear_search_range=0.25, angular_search_range=0.06, linear_step=0.025, angular_step=0.005, grid_resolution=0.05)
ODOM_SIGMA = (0.03, 0.03, 0.01)       # per-step noise of the odometry increment (forward, lateral, yaw)


def compose(p, d):
    """pose p followed by the robot-frame increment d"""
    c, s = np.cos(p[2]), np.sin(p[2])
    return np.array([p[0] + c * d[0] - s * d[1], p[1] + s * d[0] + c * d[1], p[2] + d[2]])


def odometry(truth, seed=3):
    """the truth's robot-frame increments with seeded N(0, ODOM_SIGMA) noise: (len(truth) - 1, 3)"""
    rng = np.random.default_rng(seed)
    t = np.asarray(truth, dtype=np.float64)
    out = []
    for k in range(1, len(t)):
        dx, dy = t[k, 0] - t[k - 1, 0], t[k, 1] - t[k - 1, 1]
        c, s = np.cos(t[k - 1, 2]), np.sin(t[k - 1, 2])
        d = np.array([c * dx + s * dy, -s * dx + c * dy, t[k, 2] - t[k - 1, 2]])
        out.append(d + rng.normal(0.0, 1.0, 3) * np.array(ODOM_SIGMA))
    return np.array(out)


def dead_reckoning(truth, odom):
    p = [np.asarray(truth[0], dtype=np.float64)]
    for d in odom:
        p.append(compose(p[-1], d))
    return np.array(p)


def scan_matched_mapping(sc, odom, fuse, set_reference, match):
    """scan 0 fused at truth[0]; then per step: predict from the last matched pose with the odometry increment, match the scan's
    finite beams against the map so far (set_reference() loads its obstacle cell centres), fuse the scan at the matched pose.
    fuse(pose, ranges) and match(qx, qy, pose) -> (x, y, yaw, score, converged).  Returns the matched poses (len(truth), 3) and
    the scores."""
    poses, scores = [np.asarray(sc.truth[0], dtype=np.float64)], []
    fuse(poses[0], sc.scans[0])
    for k in range(1, len(sc.truth)):
        pred = compose(poses[-1], odom[k - 1])
        set_reference()
        qx, qy = scan_points(sc.scans[k], sc.ANGLE_MIN, sc.ANGLE_INC)
        r = match(qx, qy, pred)
        poses.append(np.array(r[:3]))
        scores.append(r[3])
        fuse(poses[-1], sc.scans[k])
    return np.array(poses), np.array(scores)


def pose_errors(sc, poses):
    """max position error and max |wrapped heading error| against the truth"""
    t = np.asarray(sc.truth)
    pos = np.hypot(poses[:, 0] - t[:, 0], poses[:, 1] - t[:, 1])
    yaw = np.abs((poses[:, 2] - t[:, 2] + np.pi) % (2.0 * np.pi) - np.pi)
    return float(pos.max()), float(yaw.max())
