"""Writes tests/golden/csm_golden.json: correlative scan matching (DESIGN §3.13) restated independently in plain Python — a dict for
the lookup table, math.exp / math.cos / math.sin (glibc), and the triple loop with the `>` / `==`-and-`<` update of
correlative_scan_match (rust_robotics_slam/src/correlative_scan_matching.rs:55-197).  Every float is stored as a hex string.

    python tests/golden/make_csm_golden.py
"""
import json
import math
import os
import random

PI = 3.14159265358979323846


def sat_i32(v):
    """Rust's `as i32`: saturating, NaN -> 0"""
    if v != v:
        return 0
    if v >= 2147483647.0:
        return 2147483647
    if v <= -2147483648.0:
        return -2147483648
    return int(v)


def rs_round(v):
    """f64::round: half away from zero (Python's round() is half to even)"""
    if v != v or math.isinf(v):
        return v
    frac, whole = math.modf(v)
    if abs(frac) >= 0.5:
        whole += math.copysign(1.0, v)
    return whole


def normalize_angle(a):
    guard = 0
    while a > PI and guard < (1 << 22):
        a -= 2.0 * PI
        guard += 1
    while a < -PI and guard < (1 << 23):
        a += 2.0 * PI
        guard += 1
    return a


def cell_index(x, y, res):
    return sat_i32(rs_round(x / res)), sat_i32(rs_round(y / res))


def build_lookup_table(rx, ry, res):
    grid = {}
    sigma = res
    R = sat_i32(math.ceil(3.0 * sigma / res))
    inv = 0.5 / (sigma * sigma)
    for x, y in zip(rx, ry):
        cx, cy = cell_index(x, y, res)
        for ix in range(cx - R, cx + R + 1):
            for iy in range(cy - R, cy + R + 1):
                gx, gy = ix * res, iy * res          # i32 as f64 * res (exact conversion)
                d2 = (gx - x) * (gx - x) + (gy - y) * (gy - y)
                w = math.exp(-d2 * inv)
                if w < 1.0e-6:
                    continue
                grid[(ix, iy)] = max(grid[(ix, iy)], w) if (ix, iy) in grid else w
    return grid, R


def score_candidate(grid, qx, qy, pose, res):
    c, s = math.cos(pose[2]), math.sin(pose[2])
    score = 0.0
    for x, y in zip(qx, qy):
        wx = c * x - s * y + pose[0]
        wy = s * x + c * y + pose[1]
        score += grid.get(cell_index(wx, wy, res), 0.0)
    return score


def offsets(rng, step):
    n = sat_i32(rs_round(rng / step))
    return [i * step for i in range(-n, n + 1)]


def match(rx, ry, qx, qy, pose, cfg):
    lr, ar, ls, as_, res = cfg
    if not rx or not qx or ls <= 0.0 or as_ <= 0.0 or res <= 0.0:
        return (pose[0], pose[1], pose[2], 0.0, False)
    grid, _ = build_lookup_table(rx, ry, res)
    best = (pose[0], pose[1], normalize_angle(pose[2]), -1.0, False)
    best_pen = math.inf
    lin, ang = offsets(lr, ls), offsets(ar, as_)
    for dx in lin:
        for dy in lin:
            for dyaw in ang:
                cand = (pose[0] + dx, pose[1] + dy, normalize_angle(pose[2] + dyaw))
                s = score_candidate(grid, qx, qy, cand, res)
                pen = dx * dx + dy * dy + dyaw * dyaw
                if s > best[3] or (s == best[3] and pen < best_pen):
                    best = (cand[0], cand[1], cand[2], s, s > 0.0)
                    best_pen = pen
    return best


FIXTURE = [(0.0, 0.0), (1.0, 0.0), (2.0, 0.0), (0.0, 1.0), (0.0, 2.0), (1.0, 1.0), (1.5, 2.0)]
DEFAULT = (1.0, 0.2, 0.1, 0.02, 0.05)


def inverse_transform(points, pose):
    c, s = math.cos(pose[2]), math.sin(pose[2])
    xs, ys = [], []
    for x, y in points:
        dx, dy = x - pose[0], y - pose[1]
        xs.append(c * dx + s * dy)
        ys.append(-s * dx + c * dy)
    return xs, ys


def cases():
    fx, fy = [p[0] for p in FIXTURE], [p[1] for p in FIXTURE]
    out = []

    def add(name, rx, ry, qx, qy, pose, cfg, table=None):
        out.append(dict(name=name, rx=rx, ry=ry, qx=qx, qy=qy, pose=list(pose), cfg=list(cfg), table=table))

    add("identity", fx, fy, fx, fy, (0.0, 0.0, 0.0), DEFAULT)
    qx, qy = inverse_transform(FIXTURE, (0.4, -0.3, 0.0))
    add("translation", fx, fy, qx, qy, (0.0, 0.0, 0.0), (0.6, 0.1, 0.1, 0.05, 0.05))
    qx, qy = inverse_transform(FIXTURE, (0.0, 0.0, 0.16))
    add("rotation", fx, fy, qx, qy, (0.0, 0.0, 0.0), (0.2, 0.3, 0.1, 0.02, 0.05))
    # the cutoff radius: R = 4 where 3 res / res rounds above 3, R = 3 where it is exactly 3; the table stored
    for res in (0.05, 0.1, 0.025, 0.2, 0.25, 0.02, 0.5, 1.0):
        add("table_res_%g" % res, [0.013, 0.3, 0.3], [-0.021, 0.11, 0.11], [0.0, 0.3], [0.0, 0.1], (0.01, -0.02, 0.1),
            (2 * res, 0.04, res, 0.02, res), table=res)
    # the reference's invalid input: yaw stays as given; zero candidates: yaw normalised, score -1
    add("invalid_empty_reference", [], [], fx, fy, (1.0, 2.0, 7.0), DEFAULT)
    add("invalid_empty_query", fx, fy, [], [], (1.0, 2.0, 7.0), DEFAULT)
    add("invalid_linear_step", fx, fy, fx, fy, (1.0, 2.0, -7.0), (1.0, 0.2, 0.0, 0.02, 0.05))
    add("invalid_angular_step", fx, fy, fx, fy, (1.0, 2.0, 7.0), (1.0, 0.2, 0.1, -0.02, 0.05))
    add("invalid_resolution", fx, fy, fx, fy, (1.0, 2.0, 7.0), (1.0, 0.2, 0.1, 0.02, 0.0))
    add("no_linear_offsets", fx, fy, fx, fy, (1.0, 2.0, 7.0), (-1.0, 0.2, 0.1, 0.02, 0.05))
    add("no_angular_offsets", fx, fy, fx, fy, (1.0, 2.0, -7.0), (1.0, -0.2, 0.1, 0.02, 0.05))
    add("half_step_rounds_away", fx, fy, fx, fy, (0.0, 0.0, 0.0), (0.25, 0.05, 0.1, 0.02, 0.05))
    # every score zero: the zero-penalty candidate (the initial pose, yaw normalised)
    add("all_zero_scores", fx, fy, [50.0, 51.0], [50.0, -50.0], (0.3, -0.2, 4.0), (0.3, 0.1, 0.1, 0.05, 0.05))
    # exact ties at equal penalty: two mirror-symmetric reference points and a query point on the axis, matched at +-dx
    add("tie_equal_penalty", [-0.2, 0.2], [0.0, 0.0], [0.0], [0.0], (0.0, 0.0, 0.0), (0.2, 0.0, 0.2, 0.02, 0.05))
    add("tie_equal_penalty_y", [0.0, 0.0], [-0.3, 0.3], [0.0], [0.0], (0.0, 0.0, 0.0), (0.3, 0.0, 0.3, 0.02, 0.1))
    # saturated query cells: the rotated point's cell saturates to i32::MAX / MIN and reads 0.0
    add("saturated_query_cells", fx, fy, fx + [1.0e300, -1.0e300], fy + [1.0e300, 5.0], (0.0, 0.0, 0.0), (0.2, 0.04, 0.1, 0.02, 0.05))
    add("duplicate_reference", fx + fx + [1.0, 1.0], fy + fy + [0.0, 0.0], fx, fy, (0.05, 0.0, 0.02), (0.2, 0.04, 0.05, 0.02, 0.05))
    add("single_reference", [0.33], [-0.41], [0.0], [0.0], (0.1, -0.2, 0.0), (0.5, 0.1, 0.05, 0.05, 0.05))
    add("large_yaw", fx, fy, fx, fy, (0.0, 0.0, 1000.0), (0.2, 0.1, 0.1, 0.02, 0.05))
    add("large_negative_yaw", fx, fy, fx, fy, (0.0, 0.0, -1234.5), (0.2, 0.1, 0.1, 0.02, 0.05))
    rnd = random.Random(7)
    rx = [rnd.uniform(-3.0, 3.0) for _ in range(40)]
    ry = [rnd.uniform(-3.0, 3.0) for _ in range(40)]
    qx, qy = inverse_transform(list(zip(rx[:30], ry[:30])), (0.23, -0.17, 0.07))
    add("random_cloud", rx, ry, qx, qy, (0.0, 0.0, 0.0), (0.3, 0.1, 0.05, 0.01, 0.05))
    return out


def h(v):
    return [h(a) for a in v] if isinstance(v, (list, tuple)) else float(v).hex()


def main():
    res = []
    for c in cases():
        r = match(c["rx"], c["ry"], c["qx"], c["qy"], c["pose"], c["cfg"])
        e = dict(name=c["name"], rx=h(c["rx"]), ry=h(c["ry"]), qx=h(c["qx"]), qy=h(c["qy"]), pose=h(c["pose"]), cfg=h(c["cfg"]),
                 result=dict(x=h(r[0]), y=h(r[1]), yaw=h(r[2]), score=h(r[3]), converged=bool(r[4])))
        if c["table"] is not None:
            grid, R = build_lookup_table(c["rx"], c["ry"], c["table"])
            e["table"] = dict(R=R, cells=sorted([[k[0], k[1], v.hex()] for k, v in grid.items()]))
        res.append(e)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csm_golden.json")
    with open(path, "w") as f:
        json.dump(dict(rule="correlative_scan_match, DESIGN §3.13", cases=res), f, separators=(",", ":"))
        f.write("\n")
    print(path, len(res), "cases")


if __name__ == "__main__":
    main()
