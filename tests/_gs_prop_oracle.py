"""ctypes access to the scan-matched proposal's oracle (tests/host/gs_prop_oracle.c, which includes gs_oracle.c unchanged), and an
independent plain-Python restatement of one particle's proposal and of one whole step on tiny grids.  Test infrastructure only."""
import ctypes as C
import math
import os
import subprocess

import numpy as np

import _assoc_oracle
import _gs_oracle as GO
import _oracle

SRC = os.path.join(_oracle.ROOT, "tests", "host", "gs_prop_oracle.c")
# pfgpu_gs_default_proposal: match range / step, lattice k / kl / ka, min_hits
PROP = dict(linear_range=0.1, linear_step=0.025, angular_range=0.05, angular_step=0.0125, half_width=1, lattice_linear_step=0.01,
            lattice_angular_step=0.005, min_hits=10)
EPS = 1e-8
_LIBS = {}


def load(libm=False):
    """the oracle library (contract math, or glibc libm with libm=True), built here on first use"""
    if libm in _LIBS:
        return _LIBS[libm]
    out = os.path.join(_oracle.ROOT, "tests", "host", "libgs_prop_oracle%s.so" % ("_libm" if libm else ""))
    deps = [SRC] + [os.path.join(_oracle.ROOT, "tests", "host", f) for f in ("gs_oracle.c", "ogm_oracle.c")] + [
        os.path.join(_oracle.ROOT, "include", f) for f in ("pf_contract_math.h", "pf_odom_math.h", "fs_ekf_math.h", "fs2_math.h",
                                                            "fs_odom_math.h", "gs_prop_math.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.run(["/usr/bin/gcc"] + _assoc_oracle.CFLAGS + (["-DPF_ORACLE_LIBM"] if libm else []) + ["-shared", "-o", out, SRC, "-lm"],
                       check=True)
    L = C.CDLL(out)
    vp, dp, sz, d, u8p = C.c_void_p, _oracle.c_dp, C.c_size_t, C.c_double, C.POINTER(C.c_uint8)
    L.orc_gs_new.argtypes, L.orc_gs_new.restype = [dp, sz, sz, dp, sz, C.c_uint64, dp], vp
    L.orc_gs_free.argtypes, L.orc_gs_free.restype = [vp], None
    L.orc_gs_step.argtypes = [vp, dp, dp, dp, sz, d, d, dp, dp]
    L.orc_gsp_step.argtypes = [vp, dp, dp, dp, sz, d, d, dp, dp, dp, dp, dp, u8p]
    L.orc_gsp_one.argtypes, L.orc_gsp_one.restype = [dp, dp, sz, sz, dp, dp, dp, dp, dp, sz, d, d, dp, dp, dp, dp, u8p], d
    L.orc_gsp_norm.argtypes, L.orc_gsp_norm.restype = [dp, dp, d, d], d
    L.orc_gs_state.argtypes, L.orc_gs_state.restype = [vp, dp, dp], None
    L.orc_gs_grid.argtypes, L.orc_gs_grid.restype = [vp, sz, dp], None
    L.orc_gs_last_indices.argtypes, L.orc_gs_last_indices.restype = [vp, C.POINTER(C.c_uint32)], sz
    L.orc_gs_info.argtypes, L.orc_gs_info.restype = [vp, dp], None
    _LIBS[libm] = L
    return L


def _u8(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint8))


def pvec(prop=None):
    """the oracle's P[8] from a proposal dict (defaults for missing keys)"""
    p = dict(PROP, **(prop or {}))
    return GO._f64([p["linear_range"], p["linear_step"], p["angular_range"], p["angular_step"], p["half_width"], p["lattice_linear_step"],
                    p["lattice_angular_step"], p["min_hits"]])


class OracleGsProp(GO.OracleGs):
    """GO.OracleGs whose steps take the proposal while `prop` is a dict, and the plain rule while it is None"""

    def __init__(self, n, start, seed=0, nth=None, libm=False, ogm=None, prop=None, **model):
        super().__init__(n, start, seed=seed, nth=nth, libm=libm, ogm=ogm, **model)
        self.L = load(libm)                 # the same orc_gs layout: gs_oracle.c is compiled into this library unchanged
        self.L.orc_gs_free(self.h)
        self.h = self.L.orc_gs_new(GO._dp(GO._cfg(self.ogm)), self.W, self.H, GO._dp(GO._model(self.model, self.nth)), self.n, int(seed),
                                   GO._dp(GO._f64(start)))
        self.prop = prop
        self.xh, self.eta, self.took = np.full((self.n, 3), np.nan), np.full(self.n, np.nan), np.zeros(self.n, dtype=bool)

    def step(self, odom_prev, odom_cur, ranges, angle_min, angle_inc, nz=None, u01=None):
        if self.prop is None:
            r = super().step(odom_prev, odom_cur, ranges, angle_min, angle_inc, nz=nz, u01=u01)
            if r is not None:
                self.xh, self.eta, self.took = np.full((self.n, 3), np.nan), np.full(self.n, np.nan), np.zeros(self.n, dtype=bool)
            return r
        r = GO._f64(ranges).ravel()
        xh, eta, took = np.empty((self.n, 3)), np.empty(self.n), np.zeros(self.n, dtype=np.uint8)
        u = None if u01 is None else GO._f64([u01])
        rc = self.L.orc_gsp_step(self.h, GO._dp(GO._f64(list(odom_prev) + list(odom_cur))), GO._dp(self.alpha), GO._dp(r), r.size,
                                 float(angle_min), float(angle_inc), GO._dp(pvec(self.prop)), GO._dp(None if nz is None else GO._f64(nz)),
                                 GO._dp(u), GO._dp(xh), GO._dp(eta), _u8(took))
        if rc < 0:
            return None
        self.xh, self.eta, self.took = xh, eta, took.astype(bool)
        return bool(rc)

    def last_proposal(self):
        return self.xh.copy(), self.eta.copy(), self.took.copy()


def one(grid, pose, odom, ranges, angle_min, angle_inc, z4, prop=None, libm=False, ogm=None, alpha=GO.ALPHA_DEFAULT, **model):
    """one particle from the C oracle: (pose (3,), weight factor, x^ (3,), eta, took)"""
    o, m = dict(GO.OGM, **(ogm or {})), dict(GO.MODEL, **model)
    g = GO._f64(grid)
    p = GO._f64(pose).copy()
    r = GO._f64(ranges).ravel()
    xh, eta, took = np.empty(3), np.empty(1), np.zeros(1, dtype=np.uint8)
    f = load(libm).orc_gsp_one(GO._dp(g), GO._dp(GO._cfg(o)), g.shape[0], g.shape[1], GO._dp(GO._model(m, 0.0)), GO._dp(p),
                               GO._dp(GO._f64(odom)), GO._dp(GO._f64(alpha)), GO._dp(r), r.size, float(angle_min), float(angle_inc),
                               GO._dp(pvec(prop)), GO._dp(GO._f64(z4)), GO._dp(xh), GO._dp(eta), _u8(took))
    return p, f, xh, float(eta[0]), bool(took[0])


def norm(odom, kl, ka, libm=False, alpha=GO.ALPHA_DEFAULT):
    return load(libm).orc_gsp_norm(GO._dp(GO._f64(odom)), GO._dp(GO._f64(alpha)), float(kl), float(ka))


# ---------------------------------------------------------------------------------------------------------------------------------
# plain-Python restatement (glibc through Python's math module): independent of the C code above
def _mul33(a, b):
    c = [0.0] * 9
    for i in range(3):
        for j in range(3):
            t = a[3 * i] * b[j]
            t = a[3 * i + 1] * b[3 + j] + t
            t = a[3 * i + 2] * b[6 + j] + t
            c[3 * i + j] = t
    return c


def _inv33(m):
    mi0 = m[4] * m[8] - m[7] * m[5]
    mi1 = m[3] * m[8] - m[6] * m[5]
    mi2 = m[3] * m[7] - m[6] * m[4]
    det = m[0] * mi0 - m[1] * mi1 + m[2] * mi2
    if det == 0.0:
        return None
    return [mi0 / det, (m[2] * m[7] - m[8] * m[1]) / det, (m[1] * m[5] - m[4] * m[2]) / det, (-mi1) / det,
            (m[0] * m[8] - m[6] * m[2]) / det, (m[2] * m[3] - m[5] * m[0]) / det, mi2 / det, (m[1] * m[6] - m[7] * m[0]) / det,
            (m[0] * m[4] - m[3] * m[1]) / det]


def _sigma(inc, s, c):
    _, t, _, sr1, st, sr2 = inc
    v = [-(t * s), c, 0.0, t * c, s, 0.0, 1.0, 0.0, 1.0]
    vt = [v[0], v[3], v[6], v[1], v[4], v[7], v[2], v[5], v[8]]
    cov = _mul33(_mul33(v, [sr1 * sr1, 0.0, 0.0, 0.0, st * st, 0.0, 0.0, 0.0, sr2 * sr2]), vt)
    for i in (0, 4, 8):
        cov[i] = cov[i] + EPS
    return cov


def _move(inc, pose, za, zb, zc):
    rot1, trans, rot2, sr1, st, sr2 = inc
    r1 = GO._normalize(rot1 - (sr1 * za if sr1 > 0.0 else 0.0))
    t = trans - (st * zb if st > 0.0 else 0.0)
    r2 = GO._normalize(rot2 - (sr2 * zc if sr2 > 0.0 else 0.0))
    x, y, yaw = pose
    a = yaw + r1
    return x + t * math.cos(a), y + t * math.sin(a), GO._normalize(yaw + GO._normalize(r1 + r2))


def np_norm(inc, kl, ka):
    s = _sigma(inc, 0.0, 1.0)
    det = s[0] * (s[4] * s[8] - s[7] * s[5]) - s[1] * (s[3] * s[8] - s[6] * s[5]) + s[2] * (s[3] * s[7] - s[6] * s[4])
    tp = 2.0 * math.pi
    return ((kl * kl) * ka) / math.sqrt(((tp * tp) * tp) * det)


def _weight_hits(grid, x, y, yaw, used, angle_min, ogm, model):
    W, H = grid.shape
    res, R = ogm["resolution"], int(model["search_radius"])
    q_out = model["z_rand"] / model["max_range"]
    wr, h = 1.0, 0
    for r, a in used:
        ang = (yaw + angle_min) + a
        cx = GO._sat_i32(math.floor((x + r * math.cos(ang)) / res + W / 2.0))
        cy = GO._sat_i32(math.floor((y + r * math.sin(ang)) / res + H / 2.0))
        win = grid[max(cx - R, 0):max(min(cx + R + 1, W), 0), max(cy - R, 0):max(min(cy + R + 1, H), 0)]
        if win.size == 0:
            q = q_out
        else:
            vals = win[~np.isnan(win)]
            l = float(vals.max()) if vals.size else -math.inf
            q = model["z_hit"] * (1.0 - 1.0 / (1.0 + (math.exp(l) if l < 709.0 else math.inf))) + q_out
            h += 1 if l > 0.0 else 0
        wr = wr * q
    return wr, h


def _index(j, nl, na):
    NL, NA = 2 * nl + 1, 2 * na + 1
    return j // (NA * NL) - nl, (j // NA) % NL - nl, j % NA - na


def _chol_sample(cov, mean, n):
    """fs2_propose_pose's tail: Cholesky (or the diagonal fallback), mean + L n, yaw wrapped"""
    w, l, ok = list(cov), [0.0] * 9, True
    for j in range(3):
        for k in range(j):
            f = -w[3 * j + k]
            for i in range(j, 3):
                w[3 * i + j] = f * w[3 * i + k] + w[3 * i + j]
        dg = w[3 * j + j]
        if dg == 0.0 or not dg >= 0.0:
            ok = False
            break
        den = math.sqrt(dg)
        w[3 * j + j] = den
        for i in range(j + 1, 3):
            w[3 * i + j] = w[3 * i + j] / den
    if ok:
        l[0], l[3], l[4], l[6], l[7], l[8] = w[0], w[3], w[4], w[6], w[7], w[8]
    else:
        for i in range(3):
            c = cov[4 * i]
            l[4 * i] = math.sqrt(c if c > 0.0 else 0.0)
    out = []
    for i in range(3):
        t = l[3 * i] * n[0]
        t = l[3 * i + 1] * n[1] + t
        t = l[3 * i + 2] * n[2] + t
        out.append(mean[i] + t)
    return out[0], out[1], GO._normalize(out[2])


def _identity_pass(pose, C):
    """fs2_propose_pose's motion model and prior with a zero control: (mean, covariance) as its arithmetic leaves them"""
    x, y, yaw = pose
    sn, cs = math.sin(yaw), math.cos(yaw)
    mean = (x + 0.0 * 0.0 * cs, y + 0.0 * 0.0 * sn, GO._normalize(yaw + 0.0 * 0.0))
    g = [1.0, 0.0, -0.0 * 0.0 * sn, 0.0, 1.0, 0.0 * 0.0 * cs, 0.0, 0.0, 1.0]
    gt = [g[0], g[3], g[6], g[1], g[4], g[7], g[2], g[5], g[8]]
    return mean, _mul33(_mul33(g, C), gt)


def np_one(grid, pose, odom, ranges, angle_min, angle_inc, z4, prop=None, ogm=None, alpha=GO.ALPHA_DEFAULT, **model):
    """one particle: (pose, weight factor, x^, eta, took), as the C oracle's orc_gsp_one"""
    o, m = dict(GO.OGM, **(ogm or {})), dict(GO.MODEL, **model)
    p = dict(PROP, **(prop or {}))
    inc = GO.np_increment(odom, alpha)
    used = GO.np_used(ranges, angle_inc, int(m["max_beams"]), m["max_range"])
    return _one(grid, tuple(pose), inc, used, angle_min, z4, p, o, m, np_norm(inc, p["lattice_linear_step"], p["lattice_angular_step"]))


def _one(grid, pose, inc, used, angle_min, z4, p, o, m, c):
    nan = float("nan")
    xh, eta = (nan, nan, nan), nan
    rot1, trans, rot2, sr1, st, sr2 = inc
    x, y, yaw = pose
    s, cc = math.sin(yaw + rot1), math.cos(yaw + rot1)
    mu = _move(inc, pose, 0.0, 0.0, 0.0)
    A = _inv33(_sigma(inc, s, cc))
    if not (sr1 == 0.0 and st == 0.0 and sr2 == 0.0) and A is not None:
        ls, as_ = p["linear_step"], p["angular_step"]
        nl, na = int(GO._round(p["linear_range"] / ls)), int(GO._round(p["angular_range"] / as_))
        best = None
        for j in range((2 * nl + 1) ** 2 * (2 * na + 1)):
            a, b, e = _index(j, nl, na)
            cand = (mu[0] + float(a) * ls, mu[1] + float(b) * ls, GO._normalize(mu[2] + float(e) * as_))
            sc, h = _weight_hits(grid, *cand, used, angle_min, o, m)
            dx, dy, dyaw = float(a) * ls, float(b) * ls, float(e) * as_
            pen = (dx * dx + dy * dy) + dyaw * dyaw
            if best is None or sc > best[0] or (sc == best[0] and pen < best[1]):
                best = (sc, pen, h, cand)
        xh = best[3]
        if best[2] >= p["min_hits"]:
            k, kl, ka = int(p["half_width"]), p["lattice_linear_step"], p["lattice_angular_step"]
            offs, tau = [], []
            for j in range((2 * k + 1) ** 3):
                a, b, e = _index(j, k, k)
                pt = (xh[0] + float(a) * kl, xh[1] + float(b) * kl, GO._normalize(xh[2] + float(e) * ka))
                Lj, _ = _weight_hits(grid, *pt, used, angle_min, o, m)
                d = (pt[0] - mu[0], pt[1] - mu[1], GO._normalize(pt[2] - mu[2]))
                t = []
                for i in range(3):
                    u = A[3 * i] * d[0]
                    u = A[3 * i + 1] * d[1] + u
                    u = A[3 * i + 2] * d[2] + u
                    t.append(u)
                q = d[0] * t[0]
                q = d[1] * t[1] + q
                q = d[2] * t[2] + q
                ex = -0.5 * q
                tau.append(Lj * (math.exp(ex) if ex < 709.0 else math.inf))
                offs.append((float(a) * kl, float(b) * kl, float(e) * ka))
            T = 0.0
            for v in tau:
                T = T + v
            eta = c * T
            if 2.2250738585072014e-308 <= eta <= 1.7976931348623157e308:
                sm = [0.0, 0.0, 0.0]
                for v, of in zip(tau, offs):
                    for i in range(3):
                        sm[i] = sm[i] + v * of[i]
                mo = [sm[i] / T for i in range(3)]
                acc = dict(((i, kk), 0.0) for i in range(3) for kk in range(i, 3))
                for v, of in zip(tau, offs):
                    u = [of[i] - mo[i] for i in range(3)]
                    vv = [v * u[i] for i in range(3)]
                    for i in range(3):
                        for kk in range(i, 3):
                            acc[(i, kk)] = acc[(i, kk)] + vv[i] * u[kk]
                Cm = [0.0] * 9
                for i in range(3):
                    for kk in range(i, 3):
                        Cm[3 * i + kk] = Cm[3 * kk + i] = acc[(i, kk)] / T
                for i in (0, 4, 8):
                    Cm[i] = Cm[i] + EPS
                start = (xh[0] + mo[0], xh[1] + mo[1], GO._normalize(xh[2] + mo[2]))
                mean, cov = _identity_pass(start, Cm)
                return _chol_sample(cov, mean, (z4[0], z4[1], z4[3])), eta, xh, eta, True
    xp = _move(inc, pose, z4[0], z4[1], z4[2])
    wr, _ = _weight_hits(grid, *xp, used, angle_min, o, m)
    return xp, wr, xh, eta, False


def np_step(state, odom, ranges, angle_min, angle_inc, nz, u01, nth, prop=None, alpha=GO.ALPHA_DEFAULT, ogm=None, **model):
    """one proposal step on state = dict(poses (n, 3), w (n,), grids (n, W, H)), in place; injected normals nz (n, 4) and resample
    draw u01.  Returns (resampled, ancestors or None, neff, copies, events, x^ (n, 3), eta (n,), took (n,)); None when refused."""
    o, m = dict(GO.OGM, **(ogm or {})), dict(GO.MODEL, **model)
    p = dict(PROP, **(prop or {}))
    inc = GO.np_increment(odom, alpha)
    used = GO.np_used(ranges, angle_inc, int(m["max_beams"]), m["max_range"])
    c = np_norm(inc, p["lattice_linear_step"], p["lattice_angular_step"])
    if not (inc[3] == 0.0 and inc[4] == 0.0 and inc[5] == 0.0):
        S = 2.0 * p["half_width"] + 1.0
        hi, q_hi = c * ((S * S) * S), m["z_hit"] + m["z_rand"] / m["max_range"]
        for _ in used:
            hi = hi * q_hi
        if not hi <= 1.7976931348623157e308:
            return None
    P, w, G = state["poses"], state["w"], state["grids"]
    n = len(w)
    XH, ETA, TOOK = np.empty((n, 3)), np.empty(n), np.zeros(n, dtype=bool)
    for i in range(n):
        pose, f, XH[i], ETA[i], TOOK[i] = _one(G[i], tuple(P[i]), inc, used, angle_min, nz[i], p, o, m, c)
        P[i] = pose
        w[i] = w[i] * f
    out = _tail(state, ranges, angle_min, angle_inc, u01, nth, o)
    return out + (XH, ETA, TOOK)


def _tail(state, ranges, angle_min, angle_inc, u01, nth, ogm):
    """normalise, N_eff, fuse and resample: GO.np_step's, unchanged"""
    P, w, G = state["poses"], state["w"], state["grids"]
    n = len(w)

    def normalise():
        s = 0.0
        for v in w:
            s += v
        if s > 0.0:
            w[:] = [v / s for v in w]
    normalise()
    s2 = 0.0
    for v in w:
        s2 += v * v
    neff = 1.0 / s2 if s2 > 0.0 else 0.0
    ev = [GO.np_fuse(G[i], P[i], ranges, angle_min, angle_inc, ogm) for i in range(n)]
    if not neff < nth:
        return False, None, neff, 0, sum(ev)
    normalise()
    cum = [0.0]
    for v in w:
        cum.append(cum[-1] + v)
    r = u01 * (1.0 / n - 0.0) + 0.0
    j, idx = 0, []
    for _ in range(n):
        while r > cum[j + 1] and j < n - 1:
            j += 1
        idx.append(j)
        r += 1.0 / n
    state["poses"] = P[idx].copy()
    state["grids"] = G[idx].copy()
    state["w"] = np.full(n, 1.0 / n)
    first = [t for t in range(n) if t == 0 or idx[t] != idx[t - 1]]
    return True, idx, neff, n - len(first), sum(ev[idx[t]] for t in first)
