#!/usr/bin/env python3
"""Golden vectors of occupancy grid mapping (the rule of include/pfgpu.h pfgpu_ogm_*, DESIGN §3.12).

Run:  python tests/golden/make_ogm_golden.py      -> tests/golden/ogm_golden.json

An independent restatement in plain Python of OccupancyGridMap::update_with_scan (rust_robotics_mapping/src/occupancy_grid_map.rs:
69-131): world_to_grid with Rust's saturating `as i32`, the round-and-clamp end cell of a beam that ends outside (round half away
from zero, written out by hand: Python's round() rounds half to even), bresenham_line's loop (:164-193), the free run, the occupied
end cell and f64::clamp; and is_occupied (:136-159).  Python floats are IEEE f64 and math.cos / math.sin / math.exp are glibc's, so
tests/host/ogm_oracle.c built with -DPF_ORACLE_LIBM must reproduce this file bit for bit (tests/test_ogm_oracle.py).
"""
import json
import math
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
I32_MAX, I32_MIN = 2147483647, -2147483648
DEFAULT = dict(resolution=0.5, width=100, height=100, prior_log_odds=0.0, occupied_log_odds=0.85, free_log_odds=-0.4, max_log_odds=5.0,
               min_log_odds=-5.0)


def hx(v):
    if isinstance(v, (list, tuple)):
        return [hx(a) for a in v]
    return float(v).hex()


def sat_i32(v):
    """Rust's `as i32` of an integral f64 (or inf / NaN)"""
    if v != v:
        return 0
    if v >= 2147483647.0:
        return I32_MAX
    if v <= -2147483648.0:
        return I32_MIN
    return int(v)


def sat_floor(v):
    """Rust's `floor() as i32`"""
    if v != v or math.isinf(v):
        return sat_i32(v)
    return sat_i32(float(math.floor(v)))


def round_away(v):
    """f64::round: half away from zero"""
    if v != v or math.isinf(v):
        return v
    t = float(math.trunc(v))
    if abs(v - t) >= 0.5:                        # v - t is exact
        t += math.copysign(1.0, v)
    return t


def clamp(l, lo, hi):
    if l < lo:
        l = lo
    if l > hi:
        l = hi
    return l


def bresenham(x0, y0, x1, y1):
    cells = []
    dx, dy = abs(x1 - x0), abs(y1 - y0)
    sx = 1 if x0 < x1 else -1
    sy = 1 if y0 < y1 else -1
    x, y, err = x0, y0, dx - dy
    while True:
        cells.append((x, y))
        if x == x1 and y == y1:
            break
        e2 = 2 * err
        if e2 > -dy:
            err -= dy
            x += sx
        if e2 < dx:
            err += dx
            y += sy
    return cells


class Ogm:
    def __init__(self, cfg):
        self.c = cfg
        self.W, self.H = cfg["width"], cfg["height"]
        self.grid = [[cfg["prior_log_odds"]] * self.H for _ in range(self.W)]

    def world_to_grid(self, x, y):
        ix = sat_floor(x / self.c["resolution"] + self.W / 2.0)
        iy = sat_floor(y / self.c["resolution"] + self.H / 2.0)
        return (ix, iy) if 0 <= ix < self.W and 0 <= iy < self.H else None

    def update_with_scan(self, x, y, yaw, ranges, angle_min, angle_inc, census=None):
        origin = self.world_to_grid(x, y)
        if origin is None:
            return
        c = self.c
        for i, r in enumerate(ranges):
            if r <= 0.0 or not math.isfinite(r):
                continue
            angle = yaw + angle_min + i * angle_inc
            ex, ey = x + r * math.cos(angle), y + r * math.sin(angle)
            end = self.world_to_grid(ex, ey)
            if end is not None:
                eix, eiy = end
            else:
                vx, vy = ex / c["resolution"] + self.W / 2.0, ey / c["resolution"] + self.H / 2.0
                eix = min(max(sat_i32(round_away(vx)), 0), self.W - 1)
                eiy = min(max(sat_i32(round_away(vy)), 0), self.H - 1)
            ray = bresenham(origin[0], origin[1], eix, eiy)
            touched = ray[:-1] + ([end] if end is not None else [])
            if census is not None:
                census[0] += len(touched)
                census[2] += int(len(set(touched)) != len(touched))
                census[3] = max(census[3], len(ray))
                for t in touched:
                    census[4][t] = census[4].get(t, 0) + 1
            for cx, cy in ray[:-1]:
                if 0 <= cx < self.W and 0 <= cy < self.H:
                    self.grid[cx][cy] = clamp(self.grid[cx][cy] + c["free_log_odds"], c["min_log_odds"], c["max_log_odds"])
            if end is not None:
                self.grid[end[0]][end[1]] = clamp(self.grid[end[0]][end[1]] + c["occupied_log_odds"], c["min_log_odds"], c["max_log_odds"])

    def mask(self, threshold):
        out = []
        for col in self.grid:
            for l in col:
                try:
                    e = math.exp(l)
                except OverflowError:
                    e = math.inf
                out.append("1" if 1.0 - 1.0 / (1.0 + e) > threshold else "0")
        return "".join(out)


def case(name, cfg, calls, thresholds=(0.5, 0.2)):
    cfg = dict(DEFAULT, **cfg)
    m = Ogm(cfg)
    census = [0, 0, 0, 0, {}]
    for poses, ranges, amin, ainc in calls:
        for p, r in zip(poses, ranges):
            m.update_with_scan(p[0], p[1], p[2], r, amin, ainc, census)
    prior = cfg["prior_log_odds"]
    changed = [[ix * m.H + iy, hx(m.grid[ix][iy])] for ix in range(m.W) for iy in range(m.H)
               if float(m.grid[ix][iy]).hex() != float(prior).hex()]
    return {"name": name, "cfg": {k: (hx(v) if isinstance(v, float) else v) for k, v in cfg.items()},
            "calls": [{"poses": [hx(list(p)) for p in poses], "ranges": [hx(list(r)) for r in ranges], "angle_min": hx(amin),
                       "angle_inc": hx(ainc)} for poses, ranges, amin, ainc in calls],
            "changed": changed, "masks": {hx(t): m.mask(t) for t in thresholds},
            "census": [census[0], max(census[4].values(), default=0), census[2], census[3]]}


def main():
    rng = np.random.default_rng(20261016)
    nan, inf = float("nan"), float("inf")
    cases = []

    def ring(B, r):
        return [[r] * B]

    # the reference's defaults: a 100 x 100 grid at 0.5 m, one 36-beam scan from the centre (a cell corner), some beams leaving
    cases.append(case("default_single", {}, [([(0.0, 0.0, 0.3)], [list(rng.uniform(0.2, 40.0, 36))], -math.pi, 2 * math.pi / 36)]))
    # 1 x N and N x 1 grids: every beam that ends outside has both coordinates rounded and clamped
    cases.append(case("one_by_n", dict(width=1, height=40, resolution=0.25),
                      [([(0.05, -2.0, 0.0), (-0.1, 3.0, 1.0)], [list(rng.uniform(0.1, 8.0, 24)), list(rng.uniform(0.1, 8.0, 24))],
                        -math.pi, 2 * math.pi / 24)]))
    cases.append(case("n_by_one", dict(width=40, height=1, resolution=0.25),
                      [([(-2.0, 0.05, 0.2), (3.0, -0.1, -1.0)], [list(rng.uniform(0.1, 8.0, 24)), list(rng.uniform(0.1, 8.0, 24))],
                        -math.pi, 2 * math.pi / 24)]))
    cases.append(case("non_square", dict(width=37, height=23, resolution=0.3),
                      [([(0.4, -0.7, 2.0), (-3.0, 1.5, -0.4), (4.9, 3.0, 3.0)], [list(rng.uniform(0.05, 9.0, 50)) for _ in range(3)],
                        -2.0, 0.08)]))
    # origins on cell edges (x / res + W / 2 integral), and on the far edge (outside: a no-op)
    edges = [(-5.0, -5.0, 0.1), (0.0, 2.5, 1.1), (4.5, -0.5, -2.0), (5.0, 0.0, 0.0), (0.0, 5.0, 0.0), (-5.0, 4.5, 2.5)]
    cases.append(case("origin_on_edges", dict(width=20, height=20, resolution=0.5),
                      [(edges, [list(rng.uniform(0.1, 12.0, 16)) for _ in edges], -math.pi, 2 * math.pi / 16)]))
    cases.append(case("origin_outside", dict(width=20, height=20, resolution=0.5),
                      [([(7.0, 0.0, 0.0), (0.0, -5.01, 0.0), (nan, 200.0, 0.0)], [[3.0] * 8] * 3, -math.pi, math.pi / 4),
                       ([(nan, 1.0, 0.4)], [[2.0, 3.0, 20.0, 1.0]], -1.0, 0.5)]))
    # special ranges: NaN, +-inf, 0, negative, subnormal, huge (the end saturates the cast)
    special = [nan, inf, -inf, 0.0, -0.0, -1.0, 5e-324, 1e-300, 1e300, 1.7e308, 3.0, 12.0]
    cases.append(case("special_ranges", dict(width=24, height=18, resolution=0.5),
                      [([(0.3, 0.2, 0.7)], [special], -math.pi, 2 * math.pi / len(special))]))
    cases.append(case("nan_yaw", dict(width=24, height=18, resolution=0.5), [([(1.3, -0.2, nan)], [[1.0, 2.0, 30.0]], 0.0, 0.1),
                                                                            ([(0.0, 0.0, 0.0)], [[2.0, 3.0]], nan, 0.1)]))
    # ends outside in x only, y only, both: the round-and-clamp end cell of both coordinates
    cases.append(case("end_outside", dict(width=30, height=20, resolution=0.5),
                      [([(0.0, 0.0, 0.0)], [[9.0, 20.0, 20.0, 7.4, 7.6]], 0.0, math.pi / 2),
                       ([(6.0, 3.0, 0.0)], [[9.2, 9.2, 20.0, 20.0]], 0.0, math.pi / 4),
                       ([(-7.3, -4.8, 0.0)], [[1.0, 1.0, 1.0, 1.0, 30.0, 0.3]], -math.pi, math.pi / 3)]))
    # zero-length rays: an end in the origin's cell (occupied only), and an end just outside that clamps to the origin (nothing)
    cases.append(case("zero_length", dict(width=10, height=10, resolution=1.0),
                      [([(0.3, 0.4, 0.0), (-4.9, 0.5, math.pi), (4.9, -4.9, -math.pi / 2)], [[0.1, 0.2], [0.2, 0.2], [0.2, 0.3]],
                        0.0, 0.01)]))
    # saturation in both orders from l = 4.9: +0.85 then -0.4 gives 4.6, -0.4 then +0.85 gives 5.0
    sat = dict(width=10, height=10, resolution=1.0, prior_log_odds=4.9)
    hit = ([(0.5, 0.5, 0.0)], [[2.0]], 0.0, 0.0)          # occupied at cell (7, 5)
    thru = ([(0.5, 0.5, 0.0)], [[3.0]], 0.0, 0.0)         # free at (5 .. 7, 5), occupied at (8, 5)
    cases.append(case("saturate_occ_then_free", sat, [hit, thru]))
    cases.append(case("saturate_free_then_occ", sat, [thru, hit]))
    cases.append(case("saturate_one_batch", sat, [([(0.5, 0.5, 0.0), (0.5, 0.5, 0.0), (-3.5, 0.5, 0.0)], [[2.0], [3.0], [1.0]], 0.0, 0.0)]))
    cases.append(case("saturate_min", dict(width=12, height=12, resolution=1.0, prior_log_odds=-4.9),
                      [([(0.5, 0.5, 0.0)] * 3, [[5.0, 5.0, 5.0, 5.0]] * 3, 0.0, math.pi / 2)]))
    cases.append(case("min_equals_max", dict(width=12, height=12, resolution=1.0, prior_log_odds=3.0, max_log_odds=1.0, min_log_odds=1.0),
                      [([(0.5, 0.5, 0.3)], [[4.0, 5.0, 30.0]], 0.0, 2.0)]))
    cases.append(case("zero_deltas_prior_outside", dict(width=12, height=12, resolution=1.0, prior_log_odds=7.5, occupied_log_odds=0.0,
                                                        free_log_odds=0.0),
                      [([(0.5, 0.5, 0.3)], [[4.0, 5.0, 30.0]], 0.0, 2.0)]))
    cases.append(case("prior_below_min", dict(width=12, height=12, resolution=1.0, prior_log_odds=-9.0),
                      [([(0.5, 0.5, 0.3)], [[4.0, 5.0, 30.0]], 0.0, 2.0)]))
    # many beams of one scan through the same cells, and the same scan repeated
    cases.append(case("same_cells_one_scan", dict(width=30, height=30, resolution=0.5),
                      [([(0.1, 0.2, 0.4)], [list(np.repeat([3.0, 5.0, 6.5, 20.0], 40))], 0.0, 0.0)]))
    sc = list(rng.uniform(0.5, 9.0, 32))
    cases.append(case("repeated_scans", dict(width=40, height=40, resolution=0.5),
                      [([(0.2, -0.3, 0.1)] * 10, [sc] * 10, -math.pi, 2 * math.pi / 32), ([(0.2, -0.3, 0.1)] * 15, [sc] * 15, -math.pi,
                                                                                            2 * math.pi / 32)]))
    # random poses and ranges over several calls of uneven sizes
    calls = []
    for S in (1, 5, 2, 9):
        poses = [tuple(rng.uniform(-9.0, 9.0, 2)) + (float(rng.uniform(-4.0, 4.0)),) for _ in range(S)]
        ranges = [list(np.where(rng.random(45) < 0.1, inf, rng.uniform(0.0, 14.0, 45))) for _ in range(S)]
        calls.append((poses, ranges, -math.pi, 2 * math.pi / 45))
    cases.append(case("random_calls", dict(width=45, height=35, resolution=0.4), calls))

    path = os.path.join(HERE, "ogm_golden.json")
    with open(path, "w") as f:
        json.dump({"cases": cases}, f, separators=(",", ":"))
    print("wrote ogm_golden.json", os.path.getsize(path), "bytes;", len(cases), "cases")


if __name__ == "__main__":
    main()
