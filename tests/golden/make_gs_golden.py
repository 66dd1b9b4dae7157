#!/usr/bin/env python3
"""Writes tests/golden/gs_golden.json: grid-based FastSLAM's arithmetic (DESIGN §3.16) pinned by the plain-Python / numpy restatement
in tests/_gs_oracle.py (np_weight, np_step: glibc through Python's math module), independent of tests/host/gs_oracle.c.

  weights  one pose against one 6 x 5 grid (random log-odds with NaN cells and cells at +-inf, poses inside, on the border and outside),
           R = 0 .. 3, all-unusable scans: w_raw and the used-beam count
  steps    whole steps on 12 x 10 grids with injected normals (za, zb, zc per slot) and resample draws: R = 0, 1, 2, every step
           resampling, never resampling, a pose outside the grid, standing still, a scan with no usable beam

Floats are stored as their IEEE bit patterns (u64); the grids of a step as the SHA-256 of their bits, slot after slot.  Run from the
repository root: python tests/golden/make_gs_golden.py"""
import hashlib
import json
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _gs_oracle as GO  # noqa: E402

OGM = dict(resolution=0.5, width=12, height=10)     # the grids of the steps
WOGM = dict(resolution=1.0, width=6, height=5)      # the grids of the weight cases


def u64(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64).ravel().tolist()


def digest(grids):
    """SHA-256 of the grids' bits, slot after slot (tests/test_gs_oracle.py hashes what an oracle returns the same way)"""
    return hashlib.sha256(np.ascontiguousarray(grids, dtype=np.float64).tobytes()).hexdigest()


def weight_cases(rng):
    out = []
    for k in range(12):
        R = k % 4
        g = rng.uniform(-5, 5, size=(6, 5))
        g[rng.uniform(size=g.shape) < 0.1] = np.nan
        if k % 5 == 0:
            g[0, 0], g[5, 4] = np.inf, -np.inf
        pose = [rng.uniform(-4, 4), rng.uniform(-3, 3), rng.uniform(-math.pi, math.pi)]
        if k % 6 == 5:
            pose[0] = 9.0                                   # outside the 6 m x 5 m grids
        B = int(rng.integers(1, 40))
        r = rng.uniform(0.2, 8.0, size=B)
        r[rng.uniform(size=B) < 0.1] = np.inf
        r[rng.uniform(size=B) < 0.05] = -1.0
        if k == 7:
            r[:] = np.nan
        model = dict(search_radius=R, max_beams=int(rng.integers(2, 40)), max_range=float(rng.choice([5.0, 30.0])))
        w, used = GO.np_weight(g, pose, r, -math.pi, 2 * math.pi / B, WOGM, **model)
        out.append(dict(grid=u64(g), pose=u64(pose), ranges=u64(r), angle_min=u64([-math.pi]), angle_inc=u64([2 * math.pi / B]),
                        model=model, w=u64([w])[0], used=used))
    return out


def step_case(rng, name, n, steps, nth, start, model, scan=None, still=False):
    W, H = OGM["width"], OGM["height"]
    st = dict(poses=np.tile(np.array(start, dtype=np.float64), (n, 1)), w=np.full(n, 1.0 / n), grids=np.zeros((n, W, H)))
    rec = []
    for t in range(steps):
        od = [0.1 * t, 0.02 * t, 0.05 * t, 0.1 * t + 0.15, 0.02 * t + 0.03, 0.05 * t + 0.08]
        if still:
            od[3:] = od[:3]
        B = 24
        r = rng.uniform(0.5, 5.0, size=B) if scan is None else np.array(scan(B), dtype=np.float64)
        nz = rng.standard_normal((n, 3))
        u01 = float(rng.uniform())
        did, idx, neff, copies, events = GO.np_step(st, od, r, -math.pi, 2 * math.pi / B, nz, u01, nth, ogm=OGM, **model)
        rec.append(dict(odom=u64(od), ranges=u64(r), nz=u64(nz), u01=u64([u01])[0], resampled=did, idx=idx, neff=u64([neff])[0],
                        copies=copies, events=events, poses=u64(st["poses"]), w=u64(st["w"]), grids=digest(st["grids"])))
    return dict(name=name, n=n, nth=nth, start=start, model=model, steps=rec)


def main():
    rng = np.random.default_rng(20261018)
    cases = [
        step_case(rng, "r1", 5, 4, 3.0, [0.2, -0.3, 0.4], dict(search_radius=1, max_beams=12)),
        step_case(rng, "r0", 4, 4, 2.5, [0.0, 0.0, 0.0], dict(search_radius=0, max_beams=8)),
        step_case(rng, "r2", 5, 3, 4.0, [1.0, 0.5, -1.0], dict(search_radius=2, max_beams=24)),
        step_case(rng, "every", 4, 3, math.inf, [0.2, 0.1, 0.0], dict(search_radius=1, max_beams=12)),
        step_case(rng, "never", 4, 3, 0.0, [0.2, 0.1, 0.0], dict(search_radius=1, max_beams=12)),
        step_case(rng, "outside", 3, 3, 2.0, [9.0, 0.0, 0.0], dict(search_radius=1, max_beams=12)),
        step_case(rng, "still", 4, 3, 3.0, [0.3, 0.3, 0.3], dict(search_radius=1, max_beams=12), still=True),
        step_case(rng, "unusable", 4, 3, 3.0, [0.3, 0.3, 0.3], dict(search_radius=1, max_beams=12),
                  scan=lambda B: [math.inf, math.nan, 0.0, -2.0] * (B // 4)),
    ]
    out = dict(ogm=OGM, weight_ogm=WOGM, weights=weight_cases(rng), cases=cases)
    with open(os.path.join(HERE, "gs_golden.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
