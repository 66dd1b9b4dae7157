"""Synthetic workloads of BASELINE.json / SURVEY.md §8(d): the CALLER side of the hot path (truth trajectory,
landmark maps, observation generation).  Pure numpy host code; produces plain arrays that are fed unchanged to
the CUDA engine and, in tests/bench baselines, to the CPU oracle.

get_observations restates the reference simulator crates/rust_robotics_slam/src/fastslam1.rs:277-299 (range gate
MAX_RANGE, d + N(0,1)*sqrt(R00), wrap(atan2 - yaw) + N(0,1)*sqrt(R11)); observation noise is input data, drawn
here from numpy's PCG64 (seed 42 convention of the reference's examples).
"""
import math

import numpy as np


def normalize_angle(a):   # fs1.rs:80-89
    while a > math.pi:
        a -= 2.0 * math.pi
    while a < -math.pi:
        a += 2.0 * math.pi
    return a


def grid_landmarks(side, pitch=10.0):
    """side x side landmarks, `pitch` metres apart, origin (0,0) (C3: side=16, C4: side=32)."""
    g = np.arange(side) * pitch
    xx, yy = np.meshgrid(g, g, indexing="ij")
    return np.stack([xx.ravel(), yy.ravel()], axis=1)


def get_observations(x_true, landmarks, rng, max_range=20.0, r00=0.5, r11=0.0305):
    """fs1.rs:277-299 -> list of (d, angle, lm_id), landmark order preserved"""
    lm = np.asarray(landmarks, dtype=np.float64).reshape(-1, 2)
    dx, dy = lm[:, 0] - x_true[0], lm[:, 1] - x_true[1]
    d = np.sqrt(dx * dx + dy * dy)
    ids = np.flatnonzero(d <= max_range)
    z = []
    for lm_id in ids:
        angle = normalize_angle(math.atan2(dy[lm_id], dx[lm_id]) - x_true[2])
        z.append((float(d[lm_id]) + rng.normal() * math.sqrt(r00), angle + rng.normal() * math.sqrt(r11), int(lm_id)))
    return z


def motion_model(x, u, dt=0.1):   # fs1.rs:70-77
    return [x[0] + u[0] * dt * math.cos(x[2]), x[1] + u[0] * dt * math.sin(x[2]), normalize_angle(x[2] + u[1] * dt)]


class FastSlamScenario:
    """C3 (side=16, start (75,75,0), u=(1.0,0.025)) / C4 (side=32, start (155,55,0), u=(1.0,0.01)) of SURVEY.md §8(d)."""

    def __init__(self, side=16, start=(75.0, 75.0, 0.0), control=(1.0, 0.025), steps=110, seed=42, max_range=20.0):
        self.landmarks = grid_landmarks(side)
        self.m = self.landmarks.shape[0]
        self.start = list(start)
        self.control = list(control)
        rng = np.random.default_rng(seed)
        x = list(start)
        self.obs = []
        self.truth = []
        for _ in range(steps):
            x = motion_model(x, control)
            self.truth.append(list(x))
            self.obs.append(get_observations(x, self.landmarks, rng, max_range=max_range))

    def mean_k(self):
        return float(np.mean([len(o) for o in self.obs]))


def c3_scenario(steps=110, seed=42):
    return FastSlamScenario(16, (75.0, 75.0, 0.0), (1.0, 0.025), steps, seed)


def c4_scenario(steps=55, seed=42):
    return FastSlamScenario(32, (155.0, 55.0, 0.0), (1.0, 0.01), steps, seed)


def bigmap_scenario(steps=110, seed=42):
    """16 384 landmarks (128 x 128 grid, 10 m pitch) with C3's 40 m circle moved to the middle of the grid: the robot sits at the
    same offset from the grid lines as in C3, so it observes the same ~12.7 landmarks per step"""
    return FastSlamScenario(128, (635.0, 595.0, 0.0), (1.0, 0.025), steps, seed)


def particles_scenario(steps=110, seed=42):
    """the particle-count sweep (bench_particles.py): 36 landmarks (6 x 6 grid, 10 m pitch); the robot drives a 20 m circle
    (u = (1.0, 0.05)) about the middle of the grid, so it sees most of the map every step"""
    return FastSlamScenario(6, (25.0, 5.0, 0.0), (1.0, 0.05), steps, seed)


class PfScenario:
    """C1: the scenario of crates/rust_robotics/examples/render_gif_particle_filter.rs:21-79 (5 landmarks, rounded
    rectangle drive, obs = max(range + N(0, 0.15), 0)); C2: 360 landmarks on a 30 m circle, u = (1.0, 0.03)."""

    def __init__(self, kind="c1", steps=300, seed=42):
        rng = np.random.default_rng(seed)
        self.dt = 0.1
        if kind == "c1":
            self.landmarks = np.array([(2.0, 2.0), (10.0, 2.0), (2.0, 8.0), (10.0, 8.0), (6.0, 5.0)])
            self.init = [5.0, 5.0, 0.0, 0.0]
            noise = 0.15
        else:
            ang = np.deg2rad(np.arange(360.0))
            self.landmarks = np.stack([30.0 * np.cos(ang), 30.0 * np.sin(ang)], axis=1)
            self.init = [0.0, 0.0, 0.0, 1.0]
            noise = 0.25
        t = list(self.init[:3])
        self.controls, self.obs = [], []
        for k in range(steps):
            if kind == "c1":
                u = (1.1, 0.0) if (k // 25) % 2 == 0 else (0.5, 0.63)
            else:
                u = (1.0, 0.03)
            t[0] += u[0] * math.cos(t[2]) * self.dt
            t[1] += u[0] * math.sin(t[2]) * self.dt
            t[2] += u[1] * self.dt
            rngd = np.hypot(t[0] - self.landmarks[:, 0], t[1] - self.landmarks[:, 1])
            d = np.maximum(rngd + rng.normal(0.0, noise, rngd.shape), 0.0)
            self.controls.append(u)
            self.obs.append(np.stack([d, self.landmarks[:, 0], self.landmarks[:, 1]], axis=1))
        self.truth = t


class KidnapScenario:
    """Config 2's world (landmarks every `pitch_deg` degrees on a 30 m circle, range noise 0.25, u = (1.0, 0.03), dt 0.1) with a
    kidnap: the robot starts at (0, 0, 0), drives `before` steps, is carried by `jump` = (dx, dy, dyaw) and drives `after` more
    steps.  truth[t] = the pose the observations of step t are taken at.  before = 0: a robot that starts at start + jump,
    the global-localisation case (init_region)."""
    REGION = (-25.0, 25.0, -25.0, 25.0)          # where a lost robot may be: the box inside the landmark circle

    def __init__(self, before=30, after=60, jump=(12.0, -9.0, 0.5), pitch_deg=1.0, seed=7):
        rng = np.random.default_rng(seed)
        ang = np.deg2rad(np.arange(0.0, 360.0, pitch_deg))
        self.landmarks = np.stack([30.0 * np.cos(ang), 30.0 * np.sin(ang)], axis=1)
        self.init = [0.0, 0.0, 0.0, 1.0]
        self.before, self.dt = before, 0.1
        t = [0.0, 0.0, 0.0] if before else [jump[0], jump[1], jump[2]]
        self.controls, self.obs, self.truth = [], [], []
        for k in range(before + after):
            if before and k == before:
                t = [t[0] + jump[0], t[1] + jump[1], t[2] + jump[2]]
            u = (1.0, 0.03)
            t[0] += u[0] * math.cos(t[2]) * self.dt
            t[1] += u[0] * math.sin(t[2]) * self.dt
            t[2] += u[1] * self.dt
            rngd = np.hypot(t[0] - self.landmarks[:, 0], t[1] - self.landmarks[:, 1])
            d = np.maximum(rngd + rng.normal(0.0, 0.25, rngd.shape), 0.0)
            self.controls.append(u)
            self.obs.append(np.ascontiguousarray(np.stack([d, self.landmarks[:, 0], self.landmarks[:, 1]], axis=1)))
            self.truth.append(list(t))

    @staticmethod
    def config(n):
        """config 2's MonteCarloLocalizationConfig arguments at n particles (fixed count): (min, max, eps, z, range, v, yaw, dt)"""
        return (n, n, 0.05, 2.326, 0.25, 0.05, 0.02, 0.1)

    def error(self, k, est):
        """position error of the estimate after step k [m]"""
        return math.hypot(est[0] - self.truth[k][0], est[1] - self.truth[k][1])


def _boxes(mask, res, boxes):
    """mark the axis-aligned boxes (x0, x1, y0, y1) [m] in a mask whose world (0, 0) is the grid centre"""
    W, H = mask.shape
    for x0, x1, y0, y1 in boxes:
        i0, i1 = int(math.floor(x0 / res + W / 2.0)), int(math.ceil(x1 / res + W / 2.0))
        j0, j1 = int(math.floor(y0 / res + H / 2.0)), int(math.ceil(y1 / res + H / 2.0))
        mask[max(i0, 0):max(i1, 0), max(j0, 0):max(j1, 0)] = True


class ScanScenario:
    """A robot with a 360-beam laser in a floor plan (the likelihood-field model, DESIGN §3.9).  The plan is 40 m x 30 m at 5 cm
    (800 x 600 cells, world (0, 0) at the grid centre): outer walls, four rooms off an open hall, doors and pillars, laid out without
    symmetry so that global localisation has one answer.  The robot starts at `start` and drives u = (1.0, 0.05) for `steps` steps
    (dt 0.1).  scans[t] = B = 360 ranges from angle_min = -pi in steps of 1 degree, ray-cast against the mask from the pose
    truth[t] (no mount offset) every res / 4, plus N(0, range_noise) from numpy's PCG64 `seed`; no obstacle within max_range: inf.
    cells > 0: the plan centred in a cells x cells grid tiled with copies of it, each copy outside the centre one with an extra
    pillar of its own (the large maps of bench_scan.py); the scans are the same, since the outer walls are closed.
    symmetric: the plan united with its point mirror (plan | plan[::-1, ::-1]), so that a pose (x, y, yaw) and its mirror
    (-x, -y, yaw + pi) see the same scan: a localisation problem with two answers (the pose hypotheses, DESIGN §3.10)."""
    RES = 0.05
    REGION = (-19.7, 19.7, -14.7, 14.7)       # the plan's interior: where a lost robot may be
    B, ANGLE_MIN, ANGLE_INC, MAX_RANGE = 360, -math.pi, math.pi / 180.0, 30.0

    @staticmethod
    def plan(res=0.05):
        W, H = int(round(40.0 / res)), int(round(30.0 / res))
        m = np.zeros((W, H), dtype=bool)
        t = 0.2                                                         # wall thickness
        walls = [(-20.0, 20.0, -15.0, -15.0 + t), (-20.0, 20.0, 15.0 - t, 15.0), (-20.0, -20.0 + t, -15.0, 15.0), (20.0 - t, 20.0, -15.0, 15.0),
                 (-6.0, -6.0 + t, -15.0, -9.0), (-6.0, -6.0 + t, -7.5, 5.0),                     # west rooms, door at y -9 .. -7.5
                 (-20.0, -14.0, 5.0, 5.0 + t), (-12.5, 2.0, 5.0, 5.0 + t), (3.5, 8.0, 5.0, 5.0 + t),  # north wall, doors
                 (8.0, 8.0 + t, 5.0, 9.0), (8.0, 8.0 + t, 10.5, 15.0),                           # north-east room
                 (6.0, 12.0, -6.0, -6.0 + t), (13.5, 20.0, -6.0, -6.0 + t),                      # south-east room
                 (-20.0, -10.0, -4.0, -4.0 + t), (-8.5, -6.0, -4.0, -4.0 + t),                   # the west rooms' partition
                 (12.0, 12.0 + t, -15.0, -10.5)]
        pillars = [(x, x + 0.4, y, y + 0.4) for x, y in ((1.5, -8.0), (-12.0, -10.0), (14.0, 1.0), (3.0, 10.0), (-15.0, 10.0),
                                                         (16.0, -11.0), (-2.5, 2.0), (5.5, -1.5), (-9.0, 0.0))]
        _boxes(m, res, walls + pillars)
        return m

    def __init__(self, steps=60, start=(-3.0, -4.0, 0.3), control=(1.0, 0.05), seed=11, range_noise=0.05, cells=0, symmetric=False):
        base = self.plan(self.RES)
        if symmetric:
            base = base | base[::-1, ::-1]
        self.obstacles = base if not cells else self.tiled(base, cells)
        self.dt = 0.1
        self.start = tuple(start)
        rng = np.random.default_rng(seed)
        t = list(start)
        self.controls, self.truth, self.scans = [], [], []
        W, H = base.shape
        for _ in range(steps):
            t[0] += control[0] * math.cos(t[2]) * self.dt
            t[1] += control[0] * math.sin(t[2]) * self.dt
            t[2] += control[1] * self.dt
            r = self._cast(base, t, rng, range_noise)
            self.controls.append(tuple(control))
            self.truth.append(list(t))
            self.scans.append(np.ascontiguousarray(r))
        assert not any(base[int(math.floor(x / self.RES + W / 2.0)), int(math.floor(y / self.RES + H / 2.0))] for x, y, _ in self.truth)
        self.region = self.REGION if not cells else (-cells * self.RES / 2.0, cells * self.RES / 2.0) * 2

    @classmethod
    def _cast(cls, base, t, rng, range_noise):
        """the B ranges seen from pose t in the plan `base`, ray-cast every res / 4, with N(0, range_noise) from rng; no hit: inf"""
        ang = cls.ANGLE_MIN + np.arange(cls.B) * cls.ANGLE_INC
        ds = np.arange(1, int(cls.MAX_RANGE / (cls.RES / 4.0)) + 1) * (cls.RES / 4.0)
        W, H = base.shape
        ex = t[0] + np.cos(t[2] + ang)[:, None] * ds[None, :]
        ey = t[1] + np.sin(t[2] + ang)[:, None] * ds[None, :]
        ix, iy = np.floor(ex / cls.RES + W / 2.0).astype(np.int64), np.floor(ey / cls.RES + H / 2.0).astype(np.int64)
        inside = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
        hit = inside & base[np.clip(ix, 0, W - 1), np.clip(iy, 0, H - 1)]
        first = np.where(hit.any(axis=1), hit.argmax(axis=1), -1)
        return np.where(first >= 0, ds[first] + rng.normal(0.0, range_noise, cls.B), np.inf)

    @staticmethod
    def tiled(base, cells):
        W, H = base.shape
        ix = (np.arange(cells) - cells // 2 + W // 2) % W
        iy = (np.arange(cells) - cells // 2 + H // 2) % H
        m = base[ix[:, None], iy[None, :]]
        tx = (np.arange(cells) - cells // 2 + W // 2) // W                # the copy each cell belongs to
        ty = (np.arange(cells) - cells // 2 + H // 2) // H
        for a in np.unique(tx):
            for b in np.unique(ty):
                if a == 0 and b == 0:
                    continue
                ca, cb = np.flatnonzero(tx == a), np.flatnonzero(ty == b)
                px, py = int((a * 7919 + b * 104729) % max(W - 100, 1)) + 50, int((a * 6271 + b * 3571) % max(H - 100, 1)) + 50
                sx, sy = ca[(ca - ca[0] >= px) & (ca - ca[0] < px + 8)], cb[(cb - cb[0] >= py) & (cb - cb[0] < py + 8)]
                m[np.ix_(sx, sy)] = True
        return m

    def scan_args(self, t):
        """(ranges, angle_min, angle_inc) of step t"""
        return self.scans[t], self.ANGLE_MIN, self.ANGLE_INC

    def error(self, k, est):
        """(position error [m], heading error [rad], wrapped) of the estimate after step k"""
        return (math.hypot(est[0] - self.truth[k][0], est[1] - self.truth[k][1]),
                abs(normalize_angle(est[2] - self.truth[k][2])))



def drive_odometry(legs, start, dt, rng, trans_drift, rot_drift, rot_bias):
    """The drive of a plan of (steps, v, yaw_rate) legs from `start` at `dt`, with wheel odometry in its own frame (starting at
    (0, 0, 0)): each step's true body-frame increment (dx, dy, dtheta), with dx and dy scaled by 1 + N(0, trans_drift) and dtheta by
    1 + N(0, rot_drift) plus N(0, rot_bias) (drawn from rng, nothing for a step that does not move), composed onto the previous
    odometry pose.  Yields, per step, the true pose, the odometry pose and the (v, yaw_rate) that reproduces the odometry step over dt."""
    t = list(start)
    o = [0.0, 0.0, 0.0]
    for n, v, w in legs:
        for _ in range(n):
            p = list(t)
            t[0] += v * math.cos(t[2]) * dt
            t[1] += v * math.sin(t[2]) * dt
            t[2] += w * dt
            c, s = math.cos(p[2]), math.sin(p[2])
            gx, gy = t[0] - p[0], t[1] - p[1]
            bx, by, bt = c * gx + s * gy, -s * gx + c * gy, t[2] - p[2]
            if bx != 0.0 or by != 0.0 or bt != 0.0:
                k = 1.0 + rng.normal(0.0, trans_drift)
                bx, by = bx * k, by * k
                bt = bt * (1.0 + rng.normal(0.0, rot_drift)) + rng.normal(0.0, rot_bias)
            co, so = math.cos(o[2]), math.sin(o[2])
            o = [o[0] + co * bx - so * by, o[1] + so * bx + co * by, o[2] + bt]
            yield list(t), list(o), (math.copysign(math.hypot(bx, by), bx) / dt, bt / dt)


def leg_phases(legs):
    """{phase: (first step, end step)} of a drive, stop, turn, reverse, drive plan"""
    ends = np.cumsum([n for n, _, _ in legs])
    return {"drive": (0, ends[0]), "stop": (ends[0], ends[1]), "turn": (ends[1], ends[2]), "reverse": (ends[2], ends[3]),
            "drive_again": (ends[3], ends[4])}


class OdomScenario(ScanScenario):
    """ScanScenario's plan and laser with wheel odometry (the odometry motion model, DESIGN §3.14).  The robot starts at `start`
    and drives a plan of (steps, v, yaw_rate) legs at dt 0.1: drive, stop for several scans, turn in place, reverse, drive.
    truth[t] and scans[t] are the pose and scan after step t (as in ScanScenario).  odom[0 .. steps] are wheel-odometry poses in
    their own frame (odom[0] = (0, 0, 0)): each step's true body-frame increment (dx, dy, dtheta), with dx and dy scaled by
    1 + N(0, trans_drift) and dtheta by 1 + N(0, rot_drift) plus N(0, rot_bias), composed onto the previous odometry pose
    (numpy PCG64 `seed`, drawn before the step's scan noise).  A robot that stands still reads exactly the same odometry.
    controls[t] = the (v, yaw_rate) that reproduces odometry step t over dt: what a caller of the velocity model would invent."""
    LEGS = ((25, 1.0, 0.05), (10, 0.0, 0.0), (15, 0.0, 1.0), (12, -0.5, 0.0), (20, 1.0, -0.05))

    def __init__(self, legs=LEGS, start=(-3.0, -4.0, 0.3), seed=13, range_noise=0.05, trans_drift=0.02, rot_drift=0.05, rot_bias=0.002):
        base = self.plan(self.RES)
        self.obstacles = base
        self.dt = 0.1
        self.start = tuple(start)
        self.region = self.REGION
        rng = np.random.default_rng(seed)
        self.truth, self.scans, self.odom, self.controls = [], [], [[0.0, 0.0, 0.0]], []
        for t, o, u in drive_odometry(legs, start, self.dt, rng, trans_drift, rot_drift, rot_bias):
            self.odom.append(o)
            self.controls.append(u)
            self.truth.append(t)
            self.scans.append(np.ascontiguousarray(self._cast(base, t, rng, range_noise)))
        W, H = base.shape
        assert not any(base[int(math.floor(x / self.RES + W / 2.0)), int(math.floor(y / self.RES + H / 2.0))] for x, y, _ in self.truth)
        self.phases = leg_phases(legs)

    @property
    def steps(self):
        return len(self.truth)

    def odom_pair(self, t):
        """(previous, current) odometry pose of step t"""
        return self.odom[t], self.odom[t + 1]


class FsOdomScenario:
    """FastSlamScenario's landmark world (a grid of landmarks 10 m apart, observed by get_observations within max_range) driven
    by wheel odometry (FastSLAM's odometry motion model, DESIGN §3.15): a plan of (steps, v, yaw_rate) legs at dt 0.1 with a
    stop, a turn in place and a reverse (drive_odometry: odometry with seeded drift, and the controls a caller of the velocity model
    would derive from it).  truth[t] and obs[t] are the pose and the observations after step t; odom[0 .. steps] the odometry poses;
    phases the step range of each leg."""
    LEGS = ((30, 1.0, 0.05), (15, 0.0, 0.0), (15, 0.0, 1.0), (15, -0.5, 0.0), (25, 1.0, -0.05))

    def __init__(self, side=8, start=(25.0, 25.0, 0.0), legs=LEGS, seed=21, max_range=20.0, trans_drift=0.02, rot_drift=0.05,
                 rot_bias=0.002):
        self.landmarks = grid_landmarks(side)
        self.m = self.landmarks.shape[0]
        self.start = list(start)
        self.dt = 0.1
        rng = np.random.default_rng(seed)
        self.truth, self.obs, self.odom, self.controls = [], [], [[0.0, 0.0, 0.0]], []
        for t, o, u in drive_odometry(legs, start, self.dt, rng, trans_drift, rot_drift, rot_bias):
            self.odom.append(o)
            self.controls.append(u)
            self.truth.append(t)
            self.obs.append(get_observations(t, self.landmarks, rng, max_range=max_range))
        self.phases = leg_phases(legs)

    @property
    def steps(self):
        return len(self.truth)

    def odom_pair(self, t):
        """(previous, current) odometry pose of step t"""
        return self.odom[t], self.odom[t + 1]
