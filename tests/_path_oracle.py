"""The path history's definition (DESIGN §3.6) restated in numpy, built only from what an engine or the CPU oracle reports after
every step: the poses (state()) and the resample ancestors (last_indices(), empty when the step did not resample).  Test
infrastructure only."""
import math

import numpy as np


class Genealogy:
    """Entries (step, poses (n, 3), parents (n,)) as the ring holds them; cap = None keeps every entry."""

    def __init__(self, cap=None):
        self.cap = cap
        self.entries = []

    def root(self, step, pose_w):
        """enable / upload / seed_map: the current poses, every parent the slot itself; the window restarts"""
        n = pose_w.shape[0]
        self.entries = [(step, np.array(pose_w[:, 1:4]), np.arange(n, dtype=np.uint32))]

    def record(self, step, pose_w, idx):
        n = pose_w.shape[0]
        par = np.asarray(idx, dtype=np.uint32) if len(idx) else np.arange(n, dtype=np.uint32)
        self.entries.append((step, np.array(pose_w[:, 1:4]), par))
        if self.cap is not None and len(self.entries) > self.cap:
            self.entries.pop(0)

    def window(self):
        return self.entries[0][0], self.entries[-1][0]

    def _tail(self, max_steps):
        return self.entries if max_steps is None else self.entries[-max_steps:]

    def path(self, g, max_steps=None):
        """(steps, slots, poses) of global slot g, oldest first"""
        ent = self._tail(max_steps)
        steps, slots, poses = [], [], []
        s = g
        for j in range(len(ent) - 1, -1, -1):
            st, P, par = ent[j]
            steps.append(st); slots.append(s); poses.append(P[s])
            s = int(par[s])
        return (np.array(steps[::-1], dtype=np.uint64), np.array(slots[::-1], dtype=np.uint32), np.array(poses[::-1]).reshape(-1, 3))

    def lineage_poses(self, max_steps=None):
        """[(step, (n, 3) poses of every current slot's lineage at that step)], oldest first"""
        ent = self._tail(max_steps)
        n = ent[-1][1].shape[0]
        s = np.arange(n)
        out = []
        for j in range(len(ent) - 1, -1, -1):
            st, P, par = ent[j]
            out.append((st, P[s]))
            s = par[s].astype(np.int64)
        return out[::-1]


class VecPaths:
    """The other definition: every particle carries a list of its past poses, cloned with the particle on a resample
    (particles[j].clone(), fs1.rs:227 / fs2.rs:317)."""

    def __init__(self, pose_w):
        self.paths = [[(0, tuple(p))] for p in pose_w[:, 1:4]]

    def restart(self, step, pose_w):
        self.paths = [[(step, tuple(p))] for p in pose_w[:, 1:4]]

    def step(self, step, pose_w, idx):
        if len(idx):
            self.paths = [list(self.paths[int(j)]) for j in idx]
        for i, p in enumerate(pose_w[:, 1:4]):
            self.paths[i].append((step, tuple(p)))


def _wrap(a):
    a = np.asarray(a, dtype=np.float64)
    return np.where(np.abs(a) <= math.pi, a, a - 2.0 * math.pi * np.rint(a / (2.0 * math.pi)))


def ref_path_estimate(gen, w, max_steps=None):
    """the genealogy smoother in float64 numpy: per step the §3.4 pose estimate of the lineage poses under the current weights w,
    yaw wrapped about the centre c_s = the lineage pose of the last slot.  -> (steps, means (L, 3), covs (L, 3, 3))"""
    W = w.sum()
    steps, means, covs = [], [], []
    for st, P in gen.lineage_poses(max_steps):
        steps.append(st)
        if not (np.isfinite(W) and W > 0):
            means.append(np.full(3, np.nan)); covs.append(np.full((3, 3), np.nan))
            continue
        c = P[-1]
        d = np.stack([P[:, 0] - c[0], P[:, 1] - c[1], _wrap(P[:, 2] - c[2])], axis=1)
        a = (w[:, None] * d).sum(axis=0) / W
        mean = c + a
        mean[2] = _wrap(mean[2])
        e = d - a
        means.append(mean); covs.append(np.einsum("i,ij,ik->jk", w, e, e) / W)
    return np.array(steps, dtype=np.uint64), np.array(means), np.array(covs)
