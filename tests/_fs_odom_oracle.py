"""ctypes access to FastSLAM's odometry-model oracle (tests/host/fs_odom_oracle.c, which includes fs2_exist_oracle.c and through it
fs2_assoc_oracle.c unchanged, and links oracle/liboracle*.so).  Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

import _assoc_oracle
import _exist_oracle
import _oracle
from _oracle import f64

SRC = os.path.join(_oracle.ROOT, "tests", "host", "fs_odom_oracle.c")
ALPHA_DEFAULT = (0.2, 0.2, 0.2, 0.2)
_LIBS = {}


def load(libm=False):
    """the oracle library (contract math, or glibc libm with libm=True), built here on first use"""
    if libm in _LIBS:
        return _LIBS[libm]
    _exist_oracle.load(libm)                # builds liboracle*.so first if needed
    dep = os.path.join(_oracle.ORACLE_DIR, "liboracle_libm.so" if libm else "liboracle.so")
    out = os.path.join(_oracle.ROOT, "tests", "host", "libfs_odom_oracle%s.so" % ("_libm" if libm else ""))
    deps = [SRC, _exist_oracle.SRC, _assoc_oracle.SRC, dep] + [os.path.join(_oracle.ROOT, d) for d in (
        "oracle/fs_state.h", "include/pf_contract_math.h", "include/pf_odom_math.h", "include/fs_ekf_math.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.run(["/usr/bin/gcc"] + _assoc_oracle.CFLAGS + (["-DPF_ORACLE_LIBM"] if libm else []) + ["-shared", "-o", out, SRC, dep, "-lm"],
                       check=True)
    L = C.CDLL(out)
    vp, dp, u64p, sz, d = C.c_void_p, _oracle.c_dp, C.POINTER(C.c_uint64), C.c_size_t, C.c_double
    L.orc_fo_increment.argtypes = [dp, dp, dp]
    L.orc_fo_prior.argtypes = [dp, dp, dp, dp, dp]
    L.orc_fo_move.argtypes = [dp, dp, dp, dp]
    L.orc_fo_pose2.argtypes = [C.POINTER(_oracle.FsConfig), dp, dp, dp, d, d, dp, dp]
    L.orc_fo_step.argtypes = [vp, dp, dp, C.POINTER(_oracle.FsObs), sz, dp, d]
    L.orc_fo_step_unknown.argtypes = [vp, vp, dp, dp, dp, sz, d, dp, d, u64p, u64p]
    L.orc_fs2_ex_new.argtypes, L.orc_fs2_ex_new.restype = [vp, d], vp
    L.orc_fs2_ex_free.argtypes, L.orc_fs2_ex_free.restype = [vp], None
    L.orc_fs2_ex_reset.argtypes, L.orc_fs2_ex_reset.restype = [vp], None
    L.orc_fs2_ex_counts.argtypes, L.orc_fs2_ex_counts.restype = [vp, vp, C.POINTER(C.c_int32)], None
    _LIBS[libm] = L
    return L


def _dp(a):
    return None if a is None else a.ctypes.data_as(_oracle.c_dp)


def _odom(odom_prev, odom_cur):
    return f64(list(odom_prev) + list(odom_cur))


def increment(odom_prev, odom_cur, alpha=ALPHA_DEFAULT, libm=False):
    """(rot1, trans, rot2, s_rot1, s_trans, s_rot2), or None when refused"""
    out = np.empty(6)
    return None if load(libm).orc_fo_increment(_dp(_odom(odom_prev, odom_cur)), _dp(f64(alpha)), _dp(out)) != 0 else out


def prior(odom_prev, odom_cur, pose3, alpha=ALPHA_DEFAULT, libm=False):
    """(mu[3], Sigma + eps I [3, 3]) of the proposal at pose3"""
    mean, cov = np.empty(3), np.empty(9)
    assert load(libm).orc_fo_prior(_dp(_odom(odom_prev, odom_cur)), _dp(f64(alpha)), _dp(f64(pose3)), _dp(mean), _dp(cov)) == 0
    return mean, cov.reshape(3, 3)


def move(odom_prev, odom_cur, pose3, n3, alpha=ALPHA_DEFAULT, libm=False):
    """FastSLAM 1.0's odometry move of pose3 under the normals n3"""
    p = f64(pose3).copy()
    assert load(libm).orc_fo_move(_dp(_odom(odom_prev, odom_cur)), _dp(f64(alpha)), _dp(f64(n3)), _dp(p)) == 0
    return p


def pose2(odom_prev, odom_cur, pose3, lm6, z, n3, alpha=ALPHA_DEFAULT, libm=False, **cfg):
    """FastSLAM 2.0's odometry pose of one particle -> (case, pose): case 0 still, 1 the move, 2 the proposal"""
    c = _oracle.FsConfig()
    _oracle.load(libm).orc_fs_default_config(C.byref(c))
    for k, v in cfg.items():
        setattr(c, k, v)
    p = f64(pose3).copy()
    kase = load(libm).orc_fo_pose2(C.byref(c), _dp(_odom(odom_prev, odom_cur)), _dp(f64(alpha)), _dp(f64(lm6)), float(z[0]), float(z[1]),
                                   _dp(f64(n3)), _dp(p))
    return kase, p


class OracleFsOdom(_assoc_oracle.OracleFS2Assoc):
    """OracleFS (variant 1 or 2) with the velocity steps of OracleFS2Assoc and the odometry steps of pfgpu_fs_step_odom /
    pfgpu_fs_step_unknown_odom, so one oracle mirrors a handle that mixes the two motion models.  Existence counters: enable_existence."""

    def __init__(self, n, m, seed=42, variant=2, libm=False, **cfg):
        super().__init__(n, m, seed=seed, libm=libm, **cfg)
        if variant != 2:
            self.L.orc_fs_set_variant(self.h, variant)
        self.variant = variant
        self.O = load(libm)
        self.alpha = f64(ALPHA_DEFAULT)
        self.ex, self.removed = None, 0

    def __del__(self):
        if getattr(self, "ex", None):
            self.O.orc_fs2_ex_free(self.ex)
            self.ex = None
        super().__del__()

    def set_odom_noise(self, alpha):
        self.alpha = f64(alpha)

    def enable_existence(self, r):
        if self.ex:
            self.O.orc_fs2_ex_free(self.ex)
        self.ex, self.removed = (self.O.orc_fs2_ex_new(self.h, float(r)) if r else None), 0

    def set_state(self, pose_w, lm=None):
        super().set_state(pose_w, lm)
        if getattr(self, "ex", None):
            self.O.orc_fs2_ex_reset(self.ex)

    def seed_map(self, *a, **kw):
        super().seed_map(*a, **kw)
        if getattr(self, "ex", None):
            self.O.orc_fs2_ex_reset(self.ex)

    def existence_counts(self):
        out = np.zeros((self.n, self.m), dtype=np.int32)
        self.O.orc_fs2_ex_counts(self.h, self.ex, out.ctypes.data_as(C.POINTER(C.c_int32)))
        return out

    def step_odom(self, odom_prev, odom_cur, obs, nz3=None, u01=0.0):
        """pfgpu_fs_step_odom (obs: (d, angle, lm_id) tuples) -> resampled"""
        arr = self.obs_array(obs)
        z = None if nz3 is None else f64(nz3)
        did = self.O.orc_fo_step(self.h, _dp(_odom(odom_prev, odom_cur)), _dp(self.alpha), arr, len(obs), _dp(z), float(u01))
        assert did >= 0
        return bool(did)

    def step_unknown_odom(self, odom_prev, odom_cur, z, gate_d2=16.0, nz3=None, u01=0.0):
        """pfgpu_fs_step_unknown_odom (z: (d, angle) pairs) -> resampled; self.counts, self.removed"""
        zz = f64(z).reshape(-1, 2)
        k = zz.shape[0]
        if k == 0:
            zz = np.zeros((1, 2))
        cnt, rem = np.zeros(3, dtype=np.uint64), C.c_uint64()
        n3 = None if nz3 is None else f64(nz3)
        did = self.O.orc_fo_step_unknown(self.h, self.ex, _dp(_odom(odom_prev, odom_cur)), _dp(self.alpha), _dp(zz), k, float(gate_d2),
                                         _dp(n3), float(u01), cnt.ctypes.data_as(C.POINTER(C.c_uint64)), C.byref(rem))
        assert did >= 0
        self.counts, self.removed = cnt, int(rem.value)
        return bool(did)
