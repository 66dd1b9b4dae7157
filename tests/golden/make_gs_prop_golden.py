#!/usr/bin/env python3
"""Writes tests/golden/gs_prop_golden.json: the scan-matched proposal of grid FastSLAM (DESIGN §3.17) pinned by the plain-Python
restatement in tests/_gs_prop_oracle.py (np_one, np_step: glibc through Python's math module), independent of
tests/host/gs_prop_oracle.c.

  particles  one particle against one 16 x 12 grid at 0.1 m with injected normals (za, zb, zc, n2): random grids, ties in the match
             (a grid of equal cells), no used beam (min_hits 0 and 1), min_hits failing, pi underflowing to the fallback (a prior
             0.1 mm wide), a turn in place (t = 0), a lattice crossing +-pi, a standstill, a pose outside the grid; the pose, the
             weight factor, x^, eta and took
  steps      whole steps on 16 x 12 grids with injected normals and resample draws (R = 0, 1; lattice k = 0, 1, 2)

Floats are stored as their IEEE bit patterns (u64); the grids of a step as the SHA-256 of their bits, slot after slot.  Run from the
repository root: python tests/golden/make_gs_prop_golden.py"""
import hashlib
import json
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _gs_prop_oracle as PO  # noqa: E402

OGM = dict(resolution=0.1, width=16, height=12)
B = 24


def u64(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64).ravel().tolist()


def digest(grids):
    return hashlib.sha256(np.ascontiguousarray(grids, dtype=np.float64).tobytes()).hexdigest()


def particle(rng, name, grid, pose, odom, ranges, prop, alpha=(0.2, 0.2, 0.2, 0.2), model=None, expect=None):
    z4 = rng.standard_normal(4)
    model = model or dict(search_radius=1, max_beams=24, max_range=5.0)
    p, f, xh, eta, took = PO.np_one(grid, pose, odom, ranges, -math.pi, 2 * math.pi / len(ranges), z4, prop=prop, ogm=OGM, alpha=alpha,
                                    **model)
    if expect is not None:
        assert expect(f, eta, took), name
    return dict(name=name, grid=u64(grid), pose=u64(pose), odom=u64(odom), ranges=u64(ranges), z4=u64(z4), prop=dict(PO.PROP, **prop),
                alpha=list(alpha), model=model, out_pose=u64(p), factor=u64([f])[0], xh=u64(xh), eta=u64([eta])[0], took=took)


def particles(rng):
    W, H = OGM["width"], OGM["height"]
    out = []
    box = lambda: rng.uniform(0.3, 0.7, B)                  # noqa: E731
    for k in range(8):
        g = rng.uniform(-3, 3, (W, H))
        out.append(particle(rng, f"random{k}", g, [rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2), rng.uniform(-3, 3)],
                            [0, 0, 0, rng.uniform(0.02, 0.15), rng.uniform(-0.03, 0.03), rng.uniform(-0.1, 0.1)], box(),
                            dict(min_hits=int(rng.integers(0, 8)), half_width=int(rng.integers(0, 3))),
                            model=dict(search_radius=int(rng.integers(0, 3)), max_beams=24, max_range=5.0)))
    out.append(particle(rng, "ties", np.ones((W, H)), [0.0, 0.0, 0.2], [0, 0, 0, 0.1, 0, 0], box(), dict(min_hits=0),
                        expect=lambda f, e, t: t))
    out.append(particle(rng, "no_beam_min0", rng.uniform(-3, 3, (W, H)), [0.0, 0.0, 0.2], [0, 0, 0, 0.1, 0, 0],
                        np.full(B, np.inf), dict(min_hits=0), expect=lambda f, e, t: t))
    out.append(particle(rng, "no_beam_min1", rng.uniform(-3, 3, (W, H)), [0.0, 0.0, 0.2], [0, 0, 0, 0.1, 0, 0],
                        np.full(B, np.inf), dict(min_hits=1), expect=lambda f, e, t: not t))
    out.append(particle(rng, "min_hits_fail", rng.uniform(-3, 3, (W, H)), [0.0, 0.0, 0.2], [0, 0, 0, 0.1, 0, 0], box(),
                        dict(min_hits=25), expect=lambda f, e, t: not t and math.isnan(e)))
    g = np.full((W, H), -1.0)
    g[2, :] = 3.0                                           # one wall: the match pulls x^ off mu
    out.append(particle(rng, "pi_underflow", g, [0.0, 0.0, math.pi], [0, 0, 0, 0.1, 0, 0], np.full(B, 0.45), dict(min_hits=1),
                        alpha=(1e-12, 1e-12, 1e-12, 1e-12), model=dict(search_radius=0, max_beams=24, max_range=5.0),
                        expect=lambda f, e, t: not t and e == 0.0))
    out.append(particle(rng, "turn_in_place", rng.uniform(-3, 3, (W, H)), [0.1, 0.0, 0.3], [0, 0, 0, 0, 0, 0.4], box(), dict(min_hits=0)))
    out.append(particle(rng, "cross_pi", np.ones((W, H)), [0.0, 0.0, math.pi - 0.004], [0, 0, 0, 0.05, 0, 0.001], box(),
                        dict(min_hits=0, half_width=2, lattice_angular_step=0.01), expect=lambda f, e, t: t))
    out.append(particle(rng, "still", rng.uniform(-3, 3, (W, H)), [0.1, 0.0, 0.3], [1, 1, 0.2, 1, 1, 0.2], box(), dict(min_hits=0),
                        expect=lambda f, e, t: not t and math.isnan(e)))
    out.append(particle(rng, "outside", rng.uniform(-3, 3, (W, H)), [9.0, 0.0, 0.3], [0, 0, 0, 0.1, 0, 0], box(), dict(min_hits=0),
                        expect=lambda f, e, t: t))
    return out


def step_case(rng, name, n, steps, nth, start, model, prop):
    W, H = OGM["width"], OGM["height"]
    st = dict(poses=np.tile(np.array(start, dtype=np.float64), (n, 1)), w=np.full(n, 1.0 / n), grids=np.zeros((n, W, H)))
    rec = []
    for t in range(steps):
        od = [0.03 * t, 0.01 * t, 0.02 * t, 0.03 * t + 0.04, 0.01 * t + 0.01, 0.02 * t + 0.03]
        r = rng.uniform(0.3, 0.7, size=B)
        nz = rng.standard_normal((n, 4))
        u01 = float(rng.uniform())
        did, idx, neff, copies, events, xh, eta, took = PO.np_step(st, od, r, -math.pi, 2 * math.pi / B, nz, u01, nth, prop=prop, ogm=OGM,
                                                                   **model)
        rec.append(dict(odom=u64(od), ranges=u64(r), nz=u64(nz), u01=u64([u01])[0], resampled=did, idx=idx, neff=u64([neff])[0],
                        copies=copies, events=events, poses=u64(st["poses"]), w=u64(st["w"]), grids=digest(st["grids"]), xh=u64(xh),
                        eta=u64(eta), took=[bool(v) for v in took]))
    return dict(name=name, n=n, nth=nth, start=start, model=model, prop=dict(PO.PROP, **prop), steps=rec)


def main():
    rng = np.random.default_rng(20261019)
    cases = [
        step_case(rng, "r1k1", 4, 4, 2.5, [0.1, -0.1, 0.3], dict(search_radius=1, max_beams=24, max_range=5.0), dict(min_hits=2)),
        step_case(rng, "r0k0", 4, 4, 2.5, [0.0, 0.0, 0.0], dict(search_radius=0, max_beams=24, max_range=5.0), dict(min_hits=1, half_width=0)),
        step_case(rng, "r1k2", 3, 3, 2.0, [0.1, 0.1, -1.0], dict(search_radius=1, max_beams=24, max_range=5.0), dict(min_hits=2, half_width=2)),
    ]
    assert any(any(s["took"]) for c in cases for s in c["steps"])
    out = dict(ogm=OGM, particles=particles(rng), cases=cases)
    with open(os.path.join(HERE, "gs_prop_golden.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
