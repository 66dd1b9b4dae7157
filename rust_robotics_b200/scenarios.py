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
