#!/usr/bin/env python3
"""Golden vectors of the beam measurement model (the rule of include/pfgpu.h pfgpu_pf_beam_* / pfgpu_pf_*_beam, DESIGN §3.11).

Run:  python tests/golden/make_beam_golden.py      -> tests/golden/beam_golden.json

An independent restatement in plain Python of the clearance table (brute force over the mask padded with a ring of obstacles),
world_to_grid's saturating cast, bresenham_line's loop (rust_robotics_mapping/src/occupancy_grid_map.rs:164-193), the expected range,
the beam rule with max readings, the factor and the beam bound.  Python floats are IEEE f64 and math.* is glibc, so
tests/host/pf_beam_oracle.c built with -DPF_ORACLE_LIBM must reproduce this file bit for bit (tests/test_beam_oracle.py).
"""
import json
import math
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
DBL_MIN, DBL_MAX = 2.2250738585072014e-308, 1.7976931348623157e308
MAX_L = 4096
CAP = 255


def hx(v):
    if isinstance(v, (list, tuple)):
        return [hx(a) for a in v]
    return float(v).hex()


def sat_floor(v):
    """Rust's `floor() as i32`"""
    if v != v:
        return 0
    if v >= 2147483647.0:
        return 2147483647
    if v <= -2147483648.0:
        return -2147483648
    return int(math.floor(v))


def bresenham(x0, y0, x1, y1):
    """bresenham_line, occupancy_grid_map.rs:164-193, as a generator"""
    dx, dy = abs(x1 - x0), abs(y1 - y0)
    sx = 1 if x0 < x1 else -1
    sy = 1 if y0 < y1 else -1
    x, y, err = x0, y0, dx - dy
    while True:
        yield x, y
        if x == x1 and y == y1:
            return
        e2 = 2 * err
        if e2 > -dy:
            err -= dy
            x += sx
        if e2 < dx:
            err += dx
            y += sy


class Map:
    def __init__(self, mask, res, sigma, z_hit, z_short, z_max, z_rand, lam, max_range, max_beams):
        self.mask = mask
        self.W, self.H = len(mask), len(mask[0])
        self.res, self.sigma, self.z_hit, self.z_short, self.z_max, self.z_rand = res, sigma, z_hit, z_short, z_max, z_rand
        self.lam, self.max_range, self.max_beams = lam, max_range, max_beams
        obst = [(ix, iy) for ix in range(-1, self.W + 1) for iy in range(-1, self.H + 1)
                if ix < 0 or iy < 0 or ix >= self.W or iy >= self.H or mask[ix][iy]]
        self.clr = [[min(CAP, min(max(abs(ix - ox), abs(iy - oy)) for ox, oy in obst)) for iy in range(self.H)] for ix in range(self.W)]
        self.coeff = 1.0 / math.sqrt(2.0 * math.pi * (sigma * sigma))
        q_rand = z_rand / max_range
        lo = min(q_rand, z_max) if z_max > 0.0 else q_rand
        hi = z_hit * self.coeff + z_short * lam + max(q_rand, z_max)
        pmin = pmax = 1.0
        self.L = 0
        for m in range(1, MAX_L + 2):
            pmin *= lo
            pmax *= hi
            if not (pmin >= DBL_MIN) or not (pmax <= DBL_MAX):
                break
            self.L = m - 1

    def cell(self, x, y):
        return sat_floor(x / self.res + float(self.W) / 2.0), sat_floor(y / self.res + float(self.H) / 2.0)

    def blocked(self, x, y):
        return x < 0 or y < 0 or x >= self.W or y >= self.H or self.mask[x][y]

    def cast(self, x, y, angle):
        x0, y0 = self.cell(x, y)
        if self.blocked(x0, y0):
            return 0.0
        x1, y1 = self.cell(x + self.max_range * math.cos(angle), y + self.max_range * math.sin(angle))
        for cx, cy in bresenham(x0, y0, x1, y1):
            if self.blocked(cx, cy):
                return self.res * math.sqrt(float((cx - x0) ** 2 + (cy - y0) ** 2))
        return self.max_range

    def beams(self, ranges, angle_inc):
        B = len(ranges)
        out = []
        if B:
            s = max(1, (B - 1) // (self.max_beams - 1))
            for i in range(0, B, s):
                r = ranges[i]
                if r != r or r <= 0.0:
                    continue
                if r >= self.max_range:
                    if not self.z_max > 0.0:
                        continue
                    r = self.max_range
                out.append((r, float(i) * angle_inc))
        return None if len(out) > self.L else out

    def weight(self, pose, beams, angle_min):
        x, y, yaw = pose
        w = 1.0
        for r, a in beams:
            z = r - self.cast(x, y, (yaw + angle_min) + a)
            q = self.z_hit * self.coeff * math.exp(-(z * z) / (2.0 * (self.sigma * self.sigma)))
            if z < 0.0:
                q = q + self.z_short * self.lam * math.exp(-(self.lam * r))
            q = q + (self.z_max if r >= self.max_range else self.z_rand / self.max_range)
            w = w * q
        return w


def case(name, mask, cfg, poses, casts, scans):
    m = Map(mask, *cfg)
    c = {"name": name, "W": m.W, "H": m.H, "mask": ["".join("1" if v else "0" for v in row) for row in mask],
         "cfg": hx(cfg[:8]) + [cfg[8]], "L": m.L, "clearance": m.clr, "poses": [hx(p) for p in poses], "casts": [], "scans": []}
    for B, amin, ainc in casts:
        rh = [[m.cast(p[0], p[1], (p[2] + amin) + float(b) * ainc) for b in range(B)] for p in poses]
        c["casts"].append({"B": B, "angle_min": hx(amin), "angle_inc": hx(ainc), "rhat": [hx(r) for r in rh]})
    for ranges, amin, ainc in scans:
        b = m.beams(ranges, ainc)
        c["scans"].append({"ranges": hx(ranges), "angle_min": hx(amin), "angle_inc": hx(ainc), "used": -1 if b is None else len(b),
                           "beams": [] if b is None else [hx(list(p)) for p in b],
                           "w": [] if b is None else [hx(m.weight(p, b, amin)) for p in poses]})
    return c, m


def main():
    rng = np.random.default_rng(20261017)
    AM = (0.2, 0.95, 0.1, 0.05, 0.05, 0.1)                 # AMCL's sigma_hit, z_hit, z_short, z_max, z_rand, lambda_short

    def cfg(res, max_range, max_beams=60, **kw):
        a = dict(zip(("sigma", "z_hit", "z_short", "z_max", "z_rand", "lam"), AM))
        a.update(kw)
        return (res, a["sigma"], a["z_hit"], a["z_short"], a["z_max"], a["z_rand"], a["lam"], max_range, max_beams)

    def poses(m_w, m_h, res, n):
        """random poses over the grid and a margin, then the adversarial ones: NaN, huge, cell edges, grid edges"""
        hw, hh = m_w * res / 2.0, m_h * res / 2.0
        p = [[float(rng.uniform(-hw - res, hw + res)), float(rng.uniform(-hh - res, hh + res)), float(rng.uniform(-math.pi, math.pi))]
             for _ in range(n)]
        return p + [[math.nan, 0.0, 0.3], [0.1 * res, 0.2 * res, math.nan], [1e300, 0.0, 0.0], [0.0, -1e300, 1.0], [0.0, 0.0, 1e300],
                    [0.0, 0.0, 0.0], [-hw, -hh, 0.7], [hw - 1e-9, hh - 1e-9, -2.4], [math.nextafter(-hw, 0.0), 0.0, math.pi],
                    [res, -res, -math.pi / 2]]

    def scan(B, rmax, max_range, amin=-1.5, ainc=None, sp=True):
        r = [float(v) for v in rng.uniform(0.05, rmax, B)]
        if sp:
            for j, v in enumerate([0.0, -1.0, math.inf, -math.inf, math.nan, max_range, math.nextafter(max_range, 0.0)]):
                r[(3 * j + 1) % B] = v
        return r, amin, ainc if ainc is not None else 3.0 / max(B - 1, 1)

    cases = []
    # 1 x N and N x 1
    mask = [[False] * 17]
    mask[0][3] = mask[0][11] = True
    cases.append(case("row_1xN", mask, cfg(0.25, 3.0), poses(1, 17, 0.25, 6), [(16, -math.pi, math.pi / 8)],
                      [scan(20, 3.0, 3.0), scan(9, 5.0, 3.0, 0.0, 0.7)])[0])
    mask = [[i == 5] for i in range(13)]
    cases.append(case("col_Nx1", mask, cfg(0.3, 4.0, 5), poses(13, 1, 0.3, 6), [(8, 0.0, math.pi / 4)], [scan(13, 4.0, 4.0), scan(40, 3.0, 4.0)])[0])
    # empty and full masks
    mask = [[False] * 9 for _ in range(11)]
    cases.append(case("empty", mask, cfg(0.5, 3.0), poses(11, 9, 0.5, 4), [(12, 0.0, math.pi / 6)], [scan(30, 4.0, 3.0)])[0])
    mask = [[True] * 7 for _ in range(4)]
    cases.append(case("full", mask, cfg(0.5, 3.0), poses(4, 7, 0.5, 4), [(6, 0.3, 1.0)], [scan(30, 4.0, 3.0)])[0])
    # rays leaving through each edge, axis-aligned rays and the |dx| = |dy| tie: an empty 21 x 21 grid, poses at cell centres
    mask = [[False] * 21 for _ in range(21)]
    mask[14][3] = mask[4][16] = True
    centres = [[0.0, 0.0, 0.0], [0.25, -0.75, 0.0], [-2.25, 1.25, 0.0], [3.75, 3.75, 0.0], [-4.75, -4.75, 0.0]]
    c, m = case("edges_axes_ties", mask, cfg(0.5, 15.0), centres, [(8, 0.0, math.pi / 4), (16, 0.1, math.pi / 8), (4, math.pi / 4, math.pi / 2)],
                [([2.0, 4.0, 9.0, 15.0, math.inf, 3.0, 20.0, 1.0], 0.0, math.pi / 4)])
    ties = 0
    for p in centres:
        x0, y0 = m.cell(p[0], p[1])
        for k in range(8):
            a = k * math.pi / 4
            x1, y1 = m.cell(p[0] + 15.0 * math.cos(a), p[1] + 15.0 * math.sin(a))
            ties += abs(x1 - x0) == abs(y1 - y0) and x1 != x0
    assert ties > 0
    cases.append(c)
    # a random map with walls: starts in walls and outside, NaN and huge poses, max readings
    mask = (rng.random((24, 18)) < 0.06).tolist()
    for i in range(24):
        mask[i][9] = mask[i][9] or (i % 7 != 3)
    cases.append(case("walls", mask, cfg(0.25, 6.0), poses(24, 18, 0.25, 14), [(24, -math.pi, math.pi / 12)],
                      [scan(361, 7.0, 6.0, -math.pi, math.pi / 180.0), scan(100, 7.0, 6.0), scan(7, 4.0, 6.0)])[0])
    # z_max = 0 (max readings unused) and z_short = 0
    cases.append(case("z_max_0", mask, cfg(0.25, 6.0, z_max=0.0), poses(24, 18, 0.25, 6), [], [scan(100, 7.0, 6.0)])[0])
    cases.append(case("z_short_0", mask, cfg(0.25, 6.0, z_short=0.0), poses(24, 18, 0.25, 6), [], [scan(100, 7.0, 6.0)])[0])
    # the beam bound: z_rand 1e-30 and z_max 0 -> a small L; a scan at L used beams and one at L + 1 (refused)
    mask = (rng.random((10, 10)) < 0.1).tolist()
    bcfg = cfg(0.5, 1.0, 100, sigma=0.3, z_hit=0.9, z_max=0.0, z_rand=1e-30)
    L = Map(mask, *bcfg).L
    cases.append(case("beam_bound", mask, bcfg, poses(10, 10, 0.5, 4), [], [([0.5] * L, 0.0, 0.1), ([0.5] * (L + 1), 0.0, 0.1)])[0])
    assert cases[-1]["scans"][0]["used"] == L and cases[-1]["scans"][1]["used"] == -1
    # the stride rule for several (B, max_beams)
    mask = (rng.random((12, 12)) < 0.1).tolist()
    for B, mb in ((1, 60), (100, 60), (361, 60), (7, 2), (64, 3), (59, 60)):
        cases.append(case(f"stride_B{B}_mb{mb}", mask, cfg(0.5, 5.0, mb), poses(12, 12, 0.5, 2), [], [scan(B, 6.0, 5.0, sp=False)])[0])
    path = os.path.join(HERE, "beam_golden.json")
    with open(path, "w") as f:
        json.dump({"cases": cases}, f, separators=(",", ":"))
    print("wrote beam_golden.json", os.path.getsize(path), "bytes;", len(cases), "cases; L of the bound case", L)


if __name__ == "__main__":
    main()
