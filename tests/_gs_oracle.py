"""ctypes access to the grid-based FastSLAM oracle (tests/host/gs_oracle.c, which includes ogm_oracle.c unchanged), and an independent
numpy restatement of its weight model and of one whole step on tiny grids.  Test infrastructure only."""
import ctypes as C
import math
import os
import subprocess

import numpy as np

import _assoc_oracle
import _oracle

SRC = os.path.join(_oracle.ROOT, "tests", "host", "gs_oracle.c")
ALPHA_DEFAULT = (0.2, 0.2, 0.2, 0.2)
OGM = dict(resolution=0.5, width=100, height=100, prior_log_odds=0.0, occupied_log_odds=0.85, free_log_odds=-0.4, max_log_odds=5.0,
           min_log_odds=-5.0)
MODEL = dict(z_hit=0.95, z_rand=0.05, max_range=30.0, max_beams=60, search_radius=1)
_LIBS = {}


def load(libm=False):
    """the oracle library (contract math, or glibc libm with libm=True), built here on first use"""
    if libm in _LIBS:
        return _LIBS[libm]
    out = os.path.join(_oracle.ROOT, "tests", "host", "libgs_oracle%s.so" % ("_libm" if libm else ""))
    deps = [SRC, os.path.join(_oracle.ROOT, "tests", "host", "ogm_oracle.c")] + [os.path.join(_oracle.ROOT, "include", f) for f in (
        "pf_contract_math.h", "pf_odom_math.h", "fs_ekf_math.h")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.run(["/usr/bin/gcc"] + _assoc_oracle.CFLAGS + (["-DPF_ORACLE_LIBM"] if libm else []) + ["-shared", "-o", out, SRC, "-lm"],
                       check=True)
    L = C.CDLL(out)
    vp, dp, sz, d = C.c_void_p, _oracle.c_dp, C.c_size_t, C.c_double
    L.orc_gs_new.argtypes, L.orc_gs_new.restype = [dp, sz, sz, dp, sz, C.c_uint64, dp], vp
    L.orc_gs_free.argtypes, L.orc_gs_free.restype = [vp], None
    L.orc_gs_step.argtypes = [vp, dp, dp, dp, sz, d, d, dp, dp]
    L.orc_gs_state.argtypes, L.orc_gs_state.restype = [vp, dp, dp], None
    L.orc_gs_grid.argtypes, L.orc_gs_grid.restype = [vp, sz, dp], None
    L.orc_gs_last_indices.argtypes, L.orc_gs_last_indices.restype = [vp, C.POINTER(C.c_uint32)], sz
    L.orc_gs_info.argtypes, L.orc_gs_info.restype = [vp, dp], None
    L.orc_gs_weight.argtypes, L.orc_gs_weight.restype = [dp, dp, sz, sz, dp, d, d, d, dp, sz, d], d
    L.orc_gs_used.argtypes, L.orc_gs_used.restype = [dp, dp, sz, d, dp], sz
    L.orc_gs_limit.argtypes, L.orc_gs_limit.restype = [d, d], C.c_uint64
    L.orc_gs_is_libm.restype = C.c_int
    _LIBS[libm] = L
    return L


def _dp(a):
    return None if a is None else a.ctypes.data_as(_oracle.c_dp)


def _f64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64))


def _cfg(ogm):
    return _f64([ogm["resolution"], ogm["prior_log_odds"], ogm["occupied_log_odds"], ogm["free_log_odds"], ogm["max_log_odds"],
                 ogm["min_log_odds"]])


def _model(model, nth):
    return _f64([model["z_hit"], model["z_rand"], model["max_range"], model["max_beams"], model["search_radius"], nth])


Info = __import__("collections").namedtuple("Info", ["neff", "resampled", "copies", "events", "used", "L", "steps"])


class OracleGs:
    """grid-based FastSLAM on the CPU: n slots, each with a full (W, H) grid"""

    def __init__(self, n, start, seed=0, nth=None, libm=False, ogm=None, **model):
        self.ogm = dict(OGM, **(ogm or {}))
        self.model = dict(MODEL, **model)
        self.n, self.W, self.H = int(n), int(self.ogm["width"]), int(self.ogm["height"])
        self.nth = float(n) / 2.0 if nth is None else float(nth)
        self.alpha = _f64(ALPHA_DEFAULT)
        self.L = load(libm)
        self.h = self.L.orc_gs_new(_dp(_cfg(self.ogm)), self.W, self.H, _dp(_model(self.model, self.nth)), self.n, int(seed), _dp(_f64(start)))

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_gs_free(self.h)
            self.h = None

    def step(self, odom_prev, odom_cur, ranges, angle_min, angle_inc, nz=None, u01=None):
        """whether it resampled; None when refused"""
        r = _f64(ranges).ravel()
        u = None if u01 is None else _f64([u01])
        rc = self.L.orc_gs_step(self.h, _dp(_f64(list(odom_prev) + list(odom_cur))), _dp(self.alpha), _dp(r), r.size, float(angle_min),
                                float(angle_inc), _dp(None if nz is None else _f64(nz)), _dp(u))
        return None if rc < 0 else bool(rc)

    def particles(self):
        p = np.empty((self.n, 3))
        self.L.orc_gs_state(self.h, _dp(p), None)
        return p

    def weights(self):
        w = np.empty(self.n)
        self.L.orc_gs_state(self.h, None, _dp(w))
        return w

    def grid(self, slot):
        g = np.empty((self.W, self.H))
        self.L.orc_gs_grid(self.h, int(slot), _dp(g))
        return g

    def last_indices(self):
        idx = np.empty(self.n, dtype=np.uint32)
        k = self.L.orc_gs_last_indices(self.h, idx.ctypes.data_as(C.POINTER(C.c_uint32)))
        return idx[:k].copy()

    def info(self):
        o = np.empty(7)
        self.L.orc_gs_info(self.h, _dp(o))
        return Info(float(o[0]), bool(o[1]), int(o[2]), int(o[3]), int(o[4]), int(o[5]), int(o[6]))


def weight(grid, pose, ranges, angle_min, angle_inc, libm=False, ogm=None, **model):
    """(w_raw, used beams) of one pose against one grid, from the C oracle"""
    o, m = dict(OGM, **(ogm or {})), dict(MODEL, **model)
    g = _f64(grid)
    r = _f64(ranges).ravel()
    pairs = np.empty(2 * max(r.size, 1))
    L = load(libm)
    mv = _model(m, 0.0)
    k = L.orc_gs_used(_dp(mv), _dp(r), r.size, float(angle_inc), _dp(pairs))
    w = L.orc_gs_weight(_dp(g), _dp(_cfg(o)), g.shape[0], g.shape[1], _dp(mv), float(pose[0]), float(pose[1]), float(pose[2]), _dp(pairs), k,
                        float(angle_min))
    return w, int(k)


# ---------------------------------------------------------------------------------------------------------------------------------
# numpy / math restatement (glibc through Python's math module): independent of the C code above
def _sat_i32(v):
    if v != v:
        return 0
    return int(max(min(v, 2147483647.0), -2147483648.0))


def _normalize(a):
    while a > math.pi:
        a -= 2.0 * math.pi
    while a < -math.pi:
        a += 2.0 * math.pi
    return a


def np_used(ranges, angle_inc, max_beams, max_range):
    B = len(ranges)
    if B == 0:
        return []
    s = max(1, (B - 1) // (max_beams - 1))
    return [(float(ranges[i]), float(i) * angle_inc) for i in range(0, B, s)
            if not (ranges[i] <= 0.0 or not math.isfinite(ranges[i]) or ranges[i] >= max_range)]


def np_weight(grid, pose, ranges, angle_min, angle_inc, ogm=None, **model):
    o, m = dict(OGM, **(ogm or {})), dict(MODEL, **model)
    W, H = grid.shape
    res, R = o["resolution"], int(m["search_radius"])
    q_out = m["z_rand"] / m["max_range"]
    x, y, yaw = pose
    used = np_used(ranges, angle_inc, int(m["max_beams"]), m["max_range"])
    wr = 1.0
    for r, a in used:
        ang = (yaw + angle_min) + a
        cx = _sat_i32(math.floor((x + r * math.cos(ang)) / res + W / 2.0))
        cy = _sat_i32(math.floor((y + r * math.sin(ang)) / res + H / 2.0))
        win = grid[max(cx - R, 0):max(min(cx + R + 1, W), 0), max(cy - R, 0):max(min(cy + R + 1, H), 0)]
        vals = win[~np.isnan(win)] if win.size else win
        if win.size == 0:
            q = q_out
        else:
            l = float(vals.max()) if vals.size else -math.inf
            e = math.exp(l) if l < 709.0 else math.inf
            q = m["z_hit"] * (1.0 - 1.0 / (1.0 + e)) + q_out
        wr = wr * q
    return wr, len(used)


def _bresenham(x0, y0, x1, y1):
    dx, dy = abs(x1 - x0), abs(y1 - y0)
    sx, sy = (1 if x0 < x1 else -1), (1 if y0 < y1 else -1)
    x, y, err, out = x0, y0, dx - dy, []
    while True:
        out.append((x, y))
        if x == x1 and y == y1:
            return out
        e2 = 2 * err
        if e2 > -dy:
            err -= dy
            x += sx
        if e2 < dx:
            err += dx
            y += sy


def np_fuse(grid, pose, ranges, angle_min, angle_inc, ogm=None):
    """update_with_scan in place; returns the cell updates"""
    o = dict(OGM, **(ogm or {}))
    W, H = grid.shape
    res = o["resolution"]
    x, y, yaw = pose

    def clamp(v):
        return o["min_log_odds"] if v < o["min_log_odds"] else (o["max_log_odds"] if v > o["max_log_odds"] else v)
    ox, oy = _sat_i32(math.floor(x / res + W / 2.0)), _sat_i32(math.floor(y / res + H / 2.0))
    if not (0 <= ox < W and 0 <= oy < H):
        return 0
    ev = 0
    for i, r in enumerate(ranges):
        if r <= 0.0 or not math.isfinite(r):
            continue
        ang = yaw + angle_min + float(i) * angle_inc
        ex, ey = x + r * math.cos(ang), y + r * math.sin(ang)
        ix, iy = _sat_i32(math.floor(ex / res + W / 2.0)), _sat_i32(math.floor(ey / res + H / 2.0))
        inside = 0 <= ix < W and 0 <= iy < H
        if not inside:
            ix = min(max(_sat_i32(_round(ex / res + W / 2.0)), 0), W - 1)
            iy = min(max(_sat_i32(_round(ey / res + H / 2.0)), 0), H - 1)
        cells = _bresenham(ox, oy, ix, iy)
        for cx, cy in cells[:-1]:
            grid[cx, cy] = clamp(grid[cx, cy] + o["free_log_odds"])
        ev += len(cells) - 1
        if inside:
            grid[ix, iy] = clamp(grid[ix, iy] + o["occupied_log_odds"])
            ev += 1
    return ev


def _round(v):
    """round half away from zero (Rust's f64::round)"""
    return math.copysign(math.floor(abs(v) + 0.5), v) if math.isfinite(v) and abs(v) < 2.0 ** 52 else v


def np_increment(odom, alpha):
    x, y, yaw, x2, y2, yaw2 = odom
    dx, dy = x2 - x, y2 - y
    trans = math.sqrt(dx * dx + dy * dy)
    rot1 = 0.0 if trans < 0.01 else _normalize(math.atan2(dy, dx) - yaw)
    rot2 = _normalize(_normalize(yaw2 - yaw) - rot1)

    def rn(a):
        return min(abs(_normalize(a)), abs(_normalize(a - math.pi)))
    n1, n2 = rn(rot1), rn(rot2)
    tt, q1, q2 = trans * trans, n1 * n1, n2 * n2
    return (rot1, trans, rot2, math.sqrt(alpha[0] * q1 + alpha[1] * tt), math.sqrt((alpha[2] * tt + alpha[3] * q1) + alpha[3] * q2),
            math.sqrt(alpha[0] * q2 + alpha[1] * tt))


def np_step(state, odom, ranges, angle_min, angle_inc, nz, u01, nth, alpha=ALPHA_DEFAULT, ogm=None, **model):
    """one step on state = dict(poses (n, 3), w (n,), grids (n, W, H)), in place; injected normals nz (n, 3) and resample draw u01.
    Returns (resampled, ancestors or None, neff, copies, events)."""
    rot1, trans, rot2, sr1, st, sr2 = np_increment(odom, alpha)
    P, w, G = state["poses"], state["w"], state["grids"]
    n = len(w)
    for i in range(n):
        za, zb, zc = nz[i]
        r1 = _normalize(rot1 - (sr1 * za if sr1 > 0.0 else 0.0))
        t = trans - (st * zb if st > 0.0 else 0.0)
        r2 = _normalize(rot2 - (sr2 * zc if sr2 > 0.0 else 0.0))
        x, y, yaw = P[i]
        a = yaw + r1
        x, y = x + t * math.cos(a), y + t * math.sin(a)
        yaw = _normalize(yaw + _normalize(r1 + r2))
        P[i] = (x, y, yaw)
        wr, _ = np_weight(G[i], P[i], ranges, angle_min, angle_inc, ogm, **model)
        w[i] = w[i] * wr

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
    ev = [np_fuse(G[i], P[i], ranges, angle_min, angle_inc, ogm) for i in range(n)]
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
