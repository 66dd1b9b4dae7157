#!/usr/bin/env python3
"""Golden vectors of the likelihood-field scan model (the rule of include/pfgpu.h pfgpu_pf_lfield_* / pfgpu_pf_*_scan, DESIGN §3.9).

Run:  python tests/golden/make_lfield_golden.py      -> tests/golden/lfield_golden.json

An independent restatement in plain Python of compute_udf (distance_map.rs:15-100, with dt_1d's final loop reading the line's input),
the factor table, the beam rule, world_to_grid's saturating cast and the scan weight.  Python floats are IEEE f64 and math.* is
glibc, so tests/host/pf_lfield_oracle.c built with -DPF_ORACLE_LIBM must reproduce this file bit for bit
(tests/test_lfield_oracle.py).
"""
import json
import math
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
INF = 1e20
DBL_MIN, DBL_MAX = 2.2250738585072014e-308, 1.7976931348623157e308
MAX_L = 4096


def hx(v):
    if isinstance(v, (list, tuple)):
        return [hx(a) for a in v]
    return float(v).hex()


def dt_1d(f):
    """distance_map.rs:15-53 on the list f; returns the output line"""
    n = len(f)
    v, z = [0] * (n + 1), [0.0] * (n + 1)
    k = 0
    z[0], z[1] = -INF, INF
    for q in range(1, n):
        vk = v[k]
        s = ((f[q] + float(q * q)) - (f[vk] + float(vk * vk))) / (2.0 * float(q) - 2.0 * float(vk))
        while s <= z[k]:
            k -= 1
            vk2 = v[k]
            s = ((f[q] + float(q * q)) - (f[vk2] + float(vk2 * vk2))) / (2.0 * float(q) - 2.0 * float(vk2))
        k += 1
        v[k] = q
        z[k] = s
        if k + 1 < n + 1:
            z[k + 1] = INF
    out = [0.0] * n
    k = 0
    for q in range(n):
        while k + 1 < n + 1 and z[k + 1] < float(q):
            k += 1
        dx = float(q) - float(v[k])
        out[q] = dx * dx + f[v[k]]
    return out


def compute_udf(mask):
    W, H = len(mask), len(mask[0])
    e = [[0.0 if mask[ix][iy] else INF for iy in range(H)] for ix in range(W)]
    e = [dt_1d(row) for row in e]
    cols = [dt_1d([e[ix][iy] for ix in range(W)]) for iy in range(H)]
    return [[math.sqrt(cols[iy][ix]) for iy in range(H)] for ix in range(W)]


class Map:
    def __init__(self, mask, res, sigma, z_hit, z_rand, max_range, max_beams):
        self.W, self.H = len(mask), len(mask[0])
        self.res, self.max_range, self.max_beams = res, max_range, max_beams
        self.q_out = z_rand / max_range
        coeff = 1.0 / math.sqrt(2.0 * math.pi * (sigma * sigma))
        self.D = compute_udf(mask)
        self.q = []
        for row in self.D:
            qr = []
            for d in row:
                t = d * res
                qr.append(z_hit * (coeff * math.exp(-(t * t) / (2.0 * (sigma * sigma)))) + self.q_out)
            self.q.append(qr)
        lo, hi = self.q_out, z_hit * coeff + self.q_out
        pmin = pmax = 1.0
        self.L = 0
        for m in range(1, MAX_L + 2):
            pmin *= lo
            pmax *= hi
            if not (pmin >= DBL_MIN) or not (pmax <= DBL_MAX):
                break
            self.L = m - 1

    def beams(self, ranges, angle_inc):
        B = len(ranges)
        out = []
        if B:
            s = max(1, (B - 1) // (self.max_beams - 1))
            for i in range(0, B, s):
                r = ranges[i]
                if r <= 0.0 or not math.isfinite(r) or r >= self.max_range:
                    continue
                out.append((r, float(i) * angle_inc))
        return None if len(out) > self.L else out

    @staticmethod
    def sat_floor(v):
        """Rust's `floor() as i32`"""
        if v != v:
            return 0
        if v >= 2147483647.0:
            return 2147483647
        if v <= -2147483648.0:
            return -2147483648
        return int(math.floor(v))

    def factor(self, ex, ey):
        ix = self.sat_floor(ex / self.res + float(self.W) / 2.0)
        iy = self.sat_floor(ey / self.res + float(self.H) / 2.0)
        if ix < 0 or ix >= self.W or iy < 0 or iy >= self.H:
            return self.q_out
        return self.q[ix][iy]

    def weight(self, pose, beams, angle_min):
        x, y, yaw = pose
        w = 1.0
        for r, a in beams:
            angle = (yaw + angle_min) + a
            w = w * self.factor(x + r * math.cos(angle), y + r * math.sin(angle))
        return w


def case(name, mask, cfg, poses, scans):
    m = Map(mask, *cfg)
    c = {"name": name, "W": m.W, "H": m.H, "mask": ["".join("1" if v else "0" for v in row) for row in mask],
         "cfg": hx(cfg[:5]) + [cfg[5]], "L": m.L, "D": [hx(r) for r in m.D], "q": [hx(r) for r in m.q], "poses": [hx(p) for p in poses],
         "scans": []}
    for ranges, amin, ainc in scans:
        b = m.beams(ranges, ainc)
        c["scans"].append({"ranges": hx(ranges), "angle_min": hx(amin), "angle_inc": hx(ainc), "used": -1 if b is None else len(b),
                           "beams": [] if b is None else [hx(list(p)) for p in b],
                           "w": [] if b is None else [hx(m.weight(p, b, amin)) for p in poses]})
    return c


def main():
    rng = np.random.default_rng(20261016)
    AM = (0.2, 0.95, 0.05, 30.0, 60)                       # AMCL's defaults after the resolution
    mr = AM[3]
    specials = [0.0, -1.0, math.inf, -math.inf, math.nan, mr, math.nextafter(mr, 0.0)]

    def poses(n, span):
        p = [[float(a) for a in rng.uniform(-span, span, 2)] + [float(rng.uniform(-math.pi, math.pi))] for _ in range(n)]
        return p + [[math.nan, 0.0, 0.3], [0.1, 0.2, math.nan], [-0.75, -0.5, 0.0], [0.0, 0.0, 0.0]]

    def scan(B, rmax, amin=-1.5, ainc=None, sp=True):
        r = [float(v) for v in rng.uniform(0.05, rmax, B)]
        if sp:
            for j, v in enumerate(specials):
                r[(3 * j + 1) % B] = v
        return r, amin, ainc if ainc is not None else 3.0 / max(B - 1, 1)

    cases = []
    mask = [[False] * 17]
    mask[0][3] = mask[0][11] = True
    cases.append(case("row_1xN", mask, (0.25,) + AM, poses(6, 2.0), [scan(20, 3.0), scan(9, 5.0, 0.0, 0.7)]))
    mask = [[i == 5] for i in range(13)]
    cases.append(case("col_Nx1", mask, (0.3, 0.4, 0.8, 0.1, 8.0, 5), poses(6, 2.0), [scan(13, 4.0), scan(40, 3.0)]))
    mask = (rng.random((9, 14)) < 0.12).tolist()
    cases.append(case("nonsquare", mask, (0.5,) + AM, poses(10, 3.0), [scan(361, 6.0, -math.pi, math.pi / 180.0), scan(100, 6.0), scan(7, 4.0)]))
    mask = [[False] * 5 for _ in range(6)]
    cases.append(case("empty", mask, (0.5,) + AM, poses(4, 2.0), [scan(30, 4.0)]))
    mask = [[True] * 7 for _ in range(4)]
    cases.append(case("full", mask, (0.5,) + AM, poses(4, 2.0), [scan(30, 4.0)]))
    mask = [[False] * 4 for _ in range(5)]                 # dt_1d's final loop must read the input line here (DESIGN §3.9)
    mask[0][0] = mask[2][3] = True
    cases.append(case("two_obstacles", mask, (1.0,) + AM, poses(4, 2.0), [scan(12, 4.0)]))
    # endpoints exactly on cell edges: W = H = 8 at res 0.5 -> edges at multiples of 0.5; yaw 0 and pi/2 beams
    mask = (rng.random((8, 8)) < 0.2).tolist()
    edge = [[0.0, 0.0, 0.0], [-1.0, -0.5, 0.0], [-2.0, 1.5, 0.0], [0.5, -2.0, 0.0], [-1.25, -1.75, 0.0]]
    cases.append(case("cell_edges", mask, (0.5,) + AM, edge, [([0.5, 1.0, 1.5, 2.0, 2.5, 3.0, 5.0, 9.0], 0.0, 0.0),
                                                          ([1.0, 2.0, 0.5, 1.5], -2.0, 0.0)]))
    # the beam bound: q_out = 1e-30 -> L = 9; a scan at L used beams and one at L + 1 (refused)
    mask = (rng.random((10, 10)) < 0.1).tolist()
    cfg = (0.5, 0.3, 0.9, 1e-30, 1.0, 100)
    L = Map(mask, *cfg).L
    cases.append(case("beam_bound", mask, cfg, poses(4, 1.0), [([0.5] * L, 0.0, 0.1), ([0.5] * (L + 1), 0.0, 0.1)]))
    # the stride rule for several (B, max_beams)
    mask = (rng.random((12, 12)) < 0.1).tolist()
    for B, mb in ((1, 60), (100, 60), (361, 60), (7, 2), (64, 3), (59, 60)):
        cases.append(case(f"stride_B{B}_mb{mb}", mask, (0.5, 0.2, 0.95, 0.05, 30.0, mb), poses(2, 2.0), [scan(B, 5.0, sp=False)]))
    assert cases[7]["scans"][0]["used"] == L and cases[7]["scans"][1]["used"] == -1
    path = os.path.join(HERE, "lfield_golden.json")
    with open(path, "w") as f:
        json.dump({"cases": cases}, f, separators=(",", ":"))
    print("wrote lfield_golden.json", os.path.getsize(path), "bytes;", len(cases), "cases; L of the bound case", L)


if __name__ == "__main__":
    main()
