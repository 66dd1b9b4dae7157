#!/usr/bin/env python3
"""Golden vectors of the odometry motion model (the rule of include/pf_odom_math.h and include/pfgpu.h pfgpu_pf_*_odom, DESIGN §3.14).

Run:  python tests/golden/make_odom_golden.py      -> tests/golden/odom_golden.json

The odometry increment and the particle move are restated here from the rule, in plain Python; the velocity predict, likelihood,
normalisation, N_eff gate and both resamplers are make_golden.py's and the recovery filter make_recovery_golden.py's (imported, not
rewritten).  The draws are fixture data (numpy PCG64): (za, zb, zc) per particle for an odometry predict, (zv, zw) for a velocity
one, injection draws only for the predicts that may inject.  Python floats are IEEE f64 and math.* is glibc, so
tests/host/pf_odom_oracle.c built with -DPF_ORACLE_LIBM must reproduce this file bit for bit (tests/test_odom_oracle.py).
"""
import json
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import (P, gauss_likelihood, hx, mcl_resample_adaptive, pf_estimate, pf_neff, pf_normalize,  # noqa: E402
                         pf_predict, pf_resample_particles)
from make_recovery_golden import Recovery, region_pose  # noqa: E402

PI = math.pi
MIN_TRANS = 0.01


def normalize(a):
    """fs_normalize_angle: subtract / add 2 pi one turn at a time (at most 2^22 / 2^23 turns)"""
    g = 0
    while a > PI and g < (1 << 22):
        a -= 2.0 * PI
        g += 1
    while a < -PI and g < (1 << 23):
        a += 2.0 * PI
        g += 1
    return a


def rot_noise(a):
    d1, d2 = abs(normalize(a)), abs(normalize(a - PI))
    return d2 if d2 < d1 else d1


def increment(o, alpha):
    """(rot1, trans, rot2, s_rot1, s_trans, s_rot2) of odometry poses o = (x, y, yaw, x', y', yaw')"""
    dx, dy = o[3] - o[0], o[4] - o[1]
    trans = math.sqrt(dx * dx + dy * dy)
    rot1 = 0.0 if trans < MIN_TRANS else normalize(math.atan2(dy, dx) - o[2])
    rot2 = normalize(normalize(o[5] - o[2]) - rot1)
    n1, n2 = rot_noise(rot1), rot_noise(rot2)
    tt, q1, q2 = trans * trans, n1 * n1, n2 * n2
    a1, a2, a3, a4 = alpha
    return (rot1, trans, rot2, math.sqrt(a1 * q1 + a2 * tt), math.sqrt((a3 * tt + a4 * q1) + a4 * q2), math.sqrt(a1 * q2 + a2 * tt))


def odom_move(ps, inc, z3):
    rot1, trans, rot2, s1, st, s2 = inc
    for p, (za, zb, zc) in zip(ps, z3):
        r1 = normalize(rot1 - (s1 * za if s1 > 0.0 else 0.0))
        t = trans - (st * zb if st > 0.0 else 0.0)
        r2 = normalize(rot2 - (s2 * zc if s2 > 0.0 else 0.0))
        a = p.yaw + r1
        c, s = math.cos(a), math.sin(a)
        p.x = p.x + t * c
        p.y = p.y + t * s
        p.yaw = p.yaw + normalize(r1 + r2)


ULP = math.ulp(MIN_TRANS)
INCREMENTS = [        # (name, odometry pair, alphas)
    ("trans_at_min", [0.0, 0.0, 0.3, MIN_TRANS, 0.0, 0.4], [0.2, 0.2, 0.2, 0.2]),
    ("trans_below_min", [0.0, 0.0, 0.3, MIN_TRANS - ULP, 0.0, 0.4], [0.2, 0.2, 0.2, 0.2]),
    ("trans_above_min", [0.0, 0.0, 0.3, MIN_TRANS + ULP, 0.0, 0.4], [0.2, 0.2, 0.2, 0.2]),
    ("pure_rotation", [2.0, -1.0, 0.5, 2.0, -1.0, 1.7], [0.1, 0.05, 0.2, 0.3]),
    ("pure_translation", [1.0, 1.0, 0.25, 1.0 + 0.4 * math.cos(0.25), 1.0 + 0.4 * math.sin(0.25), 0.25], [0.05, 0.1, 0.1, 0.02]),
    ("reversing", [5.0, 3.0, 0.7, 5.0 - 0.3 * math.cos(0.7), 3.0 - 0.3 * math.sin(0.7), 0.72], [0.2, 0.2, 0.2, 0.2]),
    ("reversing_exact_pi", [0.0, 0.0, 0.0, -0.5, 0.0, 0.0], [0.2, 0.2, 0.2, 0.2]),
    ("yaw_crosses_pi", [-3.0, 4.0, 3.1, -2.9, 4.02, -3.1], [0.2, 0.2, 0.2, 0.2]),
    ("yaw_crosses_minus_pi", [-3.0, 4.0, -3.12, -3.05, 3.98, 3.13], [0.2, 0.2, 0.2, 0.2]),
    ("alphas_zero", [1.0, 2.0, 0.1, 1.3, 2.2, 0.5], [0.0, 0.0, 0.0, 0.0]),
    ("no_motion", [7.5, -2.25, 1.0, 7.5, -2.25, 1.0], [0.2, 0.2, 0.2, 0.2]),
    ("odometry_yaw_unwrapped", [0.0, 0.0, 40.0, 0.2, 0.1, 40.3], [0.2, 0.2, 0.2, 0.2]),
]
LMS = [(2.0, 2.0), (10.0, 2.0), (2.0, 8.0), (10.0, 8.0), (6.0, 5.0)]


def predict_case(rng, name, o, alpha):
    n = 16
    ps = [P(rng.uniform(-5, 5), rng.uniform(-5, 5), rng.uniform(-3.0, 3.0), rng.uniform(-1, 1), 1.0 / n) for _ in range(n)]
    ps[0].yaw, ps[1].yaw, ps[2].yaw = 1.0e3, -57.0, 2.5e6       # particle yaw far outside +-pi
    init = [hx(p.row()) for p in ps]
    z3 = rng.normal(size=(n, 3)).tolist()
    inc = increment(o, alpha)
    odom_move(ps, inc, z3)
    return {"name": name, "odom": hx(o), "alpha": hx(alpha), "inc": hx(list(inc)), "init": init, "z3": [hx(z) for z in z3],
            "particles": [hx(p.row()) for p in ps]}


def odom_path(T, start=(5.0, 5.0, 0.0)):
    """a drive with a stop, a turn in place and a reverse: truth poses T + 1 and odometry with a small drift"""
    truth, x = [list(start)], list(start)
    for t in range(T):
        if t % 7 in (3, 4):
            v, w = 0.0, 0.0                                 # stop
        elif t % 7 == 5:
            v, w = 0.0, 0.8                                 # turn in place
        elif t % 7 == 6:
            v, w = -0.6, 0.0                                # reverse
        else:
            v, w = 1.0, 0.1
        x = [x[0] + v * math.cos(x[2]) * 0.1, x[1] + v * math.sin(x[2]) * 0.1, x[2] + w * 0.1]
        truth.append(list(x))
    odom = [[p[0] * 1.01 + 0.3, p[1] * 0.99 - 0.2, p[2] * 1.02] for p in truth]     # a scaled, shifted odometry frame
    return truth, odom


def filter_case(rng, name, mode, n, T, alpha, sigma, sv=0.3, sw=0.1, dt=0.1, thr=0.5, nmax=None, eps=0.05, z=2.326, rec=None,
                velocity_at=()):
    """PF (mode 0) or MCL (mode 1) steps on the landmark world; odometry steps, or velocity steps at `velocity_at`"""
    nmax = nmax or n
    truth, odom = odom_path(T)
    r = Recovery(*rec) if rec else None
    ps = [P(5.0 + rng.uniform(-1, 1), 5.0 + rng.uniform(-1, 1), rng.uniform(-0.25, 0.25), rng.uniform(-0.5, 0.5), 1.0 / n) for _ in range(n)]
    case = {"name": name, "mode": mode, "n": n, "nmax": nmax, "threshold": hx(thr), "eps": hx(eps), "z": hx(z), "sv": hx(sv), "sw": hx(sw),
            "sigma": hx(sigma), "dt": hx(dt), "alpha": hx(alpha), "init": [hx(p.row()) for p in ps], "steps": []}
    if rec:
        case["a_slow"], case["a_fast"], case["region"] = hx(rec[0]), hx(rec[1]), hx(rec[2])
    for t in range(T):
        tx, ty = truth[t + 1][0], truth[t + 1][1]
        far = rec is not None and t in (4, 5, 6)
        obs = [[1.0e4 if far else max(math.hypot(tx - lx, ty - ly) + rng.normal(0, 0.1), 0.0), lx, ly] for lx, ly in LMS]
        cur = len(ps)
        step = {"obs": [hx(o) for o in obs]}
        inj4 = []
        if r is not None:
            if r.armed and r.p > 0.0:
                inj4 = rng.uniform(size=(cur, 4)).tolist()
                for i, p in enumerate(ps):
                    if inj4[i][0] < r.p:
                        p.x, p.y, p.yaw = region_pose(rec[2], inj4[i][1], inj4[i][2], inj4[i][3])
                        p.v = 0.0
            r.armed = False
        step["inj4"] = [hx(a) for a in inj4]
        if t in velocity_at:
            u = [1.0, 0.1]
            zv, zw = rng.normal(size=cur).tolist(), rng.normal(size=cur).tolist()
            pf_predict(ps, u, zv, zw, sv, sw, dt)
            step.update({"u": hx(u), "zv": hx(zv), "zw": hx(zw)})
        else:
            o = odom[t] + odom[t + 1]
            z3 = rng.normal(size=(cur, 3)).tolist()
            odom_move(ps, increment(o, alpha), z3)
            step.update({"odom": hx(o), "z3": [hx(a) for a in z3]})
        for p in ps:
            w = 1.0
            for (d_obs, lx, ly) in obs:
                dx, dy = p.x - lx, p.y - ly
                w *= gauss_likelihood(d_obs - math.sqrt(dx * dx + dy * dy), sigma)
            p.w = w
        S = 0.0
        for p in ps:
            S += p.w
        if r is not None:
            r.filter(S, len(ps))
        pf_normalize(ps)
        rs = rng.uniform(size=n if mode == 0 else nmax).tolist()
        if mode == 0:
            did = pf_neff(ps) < float(n) * thr
            idxs = []
            if did:
                ps, idxs = pf_resample_particles(ps, n, rs)
        else:
            ps, idxs = mcl_resample_adaptive(ps, n, nmax, eps, z, rs)
            did = True
        if r is not None:
            r.armed = did
        step.update({"r": hx(rs), "did_resample": bool(did), "indices": idxs, "count": len(ps), "est": hx(pf_estimate(ps))})
        case["steps"].append(step)
    case["particles"] = [hx(p.row()) for p in ps]
    return case


def main():
    rng = np.random.default_rng(20261017)
    preds = [predict_case(rng, name, o, a) for name, o, a in INCREMENTS]
    cases = [
        filter_case(rng, "pf_gate_closed_steps", 0, 24, 10, [0.05, 0.05, 0.05, 0.05], 0.35, thr=0.5),
        filter_case(rng, "mcl_kld", 1, 12, 10, [0.2, 0.2, 0.2, 0.2], 0.5, nmax=40, eps=0.5),
        filter_case(rng, "mcl_recovery", 1, 16, 12, [0.1, 0.1, 0.1, 0.1], 0.5, rec=(0.1, 0.6, [0.0, 12.0, 0.0, 10.0])),
        filter_case(rng, "pf_mixed_velocity", 0, 20, 10, [0.2, 0.1, 0.2, 0.1], 0.5, thr=0.6, velocity_at=(2, 3, 7)),
    ]
    path = os.path.join(HERE, "odom_golden.json")
    with open(path, "w") as f:
        json.dump({"predicts": preds, "cases": cases}, f, separators=(",", ":"))
    for c in cases:
        print(c["name"], "resampled", [int(s["did_resample"]) for s in c["steps"]], "count", [s["count"] for s in c["steps"]])
    print("wrote odom_golden.json", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
