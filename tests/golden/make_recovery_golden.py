#!/usr/bin/env python3
"""Golden vectors of augmented MCL on the PF / MCL step (the rule of include/pfgpu.h pfgpu_pf_recovery_*, DESIGN §3.8).

Run:  python tests/golden/make_recovery_golden.py      -> tests/golden/recovery_golden.json

Predict, likelihood, normalisation, N_eff gate and both resamplers are make_golden.py's (imported, not rewritten); stated here are
the filter, the injection and init_region.  The draws are fixture data (numpy PCG64); injection draws (a0, a1, b0, b1) only for the
predicts that may inject.  Python floats are IEEE f64 and math.* is glibc, so tests/host/pf_recovery_oracle.c built with
-DPF_ORACLE_LIBM must reproduce this file bit for bit (tests/test_recovery_oracle.py).
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


class Recovery:
    def __init__(self, a_slow, a_fast, region):
        self.a_slow, self.a_fast, self.region = a_slow, a_fast, region
        self.w_slow = self.w_fast = self.p = 0.0
        self.armed = False

    def filter(self, S, n):
        if math.isfinite(S):
            w_avg = S / float(n)
            self.w_slow = self.w_slow + self.a_slow * (w_avg - self.w_slow)
            self.w_fast = self.w_fast + self.a_fast * (w_avg - self.w_fast)
        p = 0.0
        if self.w_slow > 0.0:
            q = self.w_fast / self.w_slow
            if math.isfinite(q):
                p = 1.0 - q
                if not p > 0.0:
                    p = 0.0
        self.p = p


def region_pose(r, fx, fy, fyaw):
    return r[0] + fx * (r[1] - r[0]), r[2] + fy * (r[3] - r[2]), fyaw * (2.0 * math.pi) - math.pi


def run_case(name, rng, mode, n, T, lms, sigma, sv, sw, a_slow, a_fast, region, thr=0.5, nmax=None, eps=0.05, z=2.326,
             start=(5.0, 5.0, 0.0), u_of=lambda t: [1.0, 0.05], kidnap=None, far_at=(), init_region=False, dt=0.1):
    """kidnap = (step, dx, dy): the truth jumps before that step's motion; far_at: steps whose observations underflow (S = 0)"""
    nmax = nmax or n
    rec = Recovery(a_slow, a_fast, region)
    case = {"name": name, "mode": mode, "n": n, "nmax": nmax, "threshold": hx(thr), "eps": hx(eps), "z": hx(z), "sv": hx(sv),
            "sw": hx(sw), "sigma": hx(sigma), "dt": hx(dt), "a_slow": hx(a_slow), "a_fast": hx(a_fast), "region": hx(region), "steps": []}
    if init_region:
        u3 = rng.uniform(size=(n, 3)).tolist()
        ps = []
        for f in u3:
            x, y, yaw = region_pose(region, *f)
            ps.append(P(x, y, yaw, 0.0, 1.0 / float(n)))
        case["init_region_u3"] = [hx(f) for f in u3]
    else:
        ps = [P(start[0] + rng.uniform(-1, 1), start[1] + rng.uniform(-1, 1), start[2] + rng.uniform(-0.25, 0.25), rng.uniform(-0.5, 0.5),
                1.0 / n) for _ in range(n)]
    case["init"] = [hx(p.row()) for p in ps]
    truth = list(start)
    for t in range(T):
        u = u_of(t)
        if kidnap and kidnap[0] == t:
            truth[0] += kidnap[1]
            truth[1] += kidnap[2]
        truth[0] += u[0] * math.cos(truth[2]) * dt
        truth[1] += u[0] * math.sin(truth[2]) * dt
        truth[2] += u[1] * dt
        obs = [[max(math.hypot(truth[0] - lx, truth[1] - ly) + rng.normal(0, 0.1), 0.0), lx, ly] for lx, ly in lms]
        if t in far_at:
            obs = [[1.0e4, lx, ly] for lx, ly in lms]
        cur = len(ps)
        zv, zw = rng.normal(size=cur).tolist(), rng.normal(size=cur).tolist()
        rs = rng.uniform(size=n if mode == 0 else nmax).tolist()
        inj4, injected = [], 0
        if rec.armed and rec.p > 0.0:                  # draws only for the predicts that may inject
            inj4 = rng.uniform(size=(cur, 4)).tolist()
            for i, p in enumerate(ps):
                if inj4[i][0] < rec.p:
                    p.x, p.y, p.yaw = region_pose(region, inj4[i][1], inj4[i][2], inj4[i][3])
                    p.v = 0.0
                    injected += 1
        rec.armed = False
        pf_predict(ps, u, zv, zw, sv, sw, dt)
        for p in ps:                                   # pf_update's likelihood loop, keeping S for the filter
            w = 1.0
            for (d_obs, lx, ly) in obs:
                dx, dy = p.x - lx, p.y - ly
                w *= gauss_likelihood(d_obs - math.sqrt(dx * dx + dy * dy), sigma)
            p.w = w
        S = 0.0
        for p in ps:
            S += p.w
        rec.filter(S, len(ps))
        pf_normalize(ps)
        if mode == 0:
            did = pf_neff(ps) < float(n) * thr
            idxs = []
            if did:
                ps, idxs = pf_resample_particles(ps, n, rs)
        else:
            ps, idxs = mcl_resample_adaptive(ps, n, nmax, eps, z, rs)
            did = True
        rec.armed = did
        case["steps"].append({"u": hx(u), "obs": [hx(o) for o in obs], "zv": hx(zv), "zw": hx(zw), "inj4": [hx(a) for a in inj4],
                              "r": hx(rs), "injected": injected, "S": hx(S), "w_slow": hx(rec.w_slow), "w_fast": hx(rec.w_fast),
                              "p": hx(rec.p), "did_resample": bool(did), "indices": idxs, "count": len(ps), "est": hx(pf_estimate(ps))})
    case["particles"] = [hx(p.row()) for p in ps]      # the final set; every step pins the estimate, indices and averages
    return case


def main():
    rng = np.random.default_rng(20261016)
    c1 = [(2.0, 2.0), (10.0, 2.0), (2.0, 8.0), (10.0, 8.0), (6.0, 5.0)]
    ring = [(10.0, 0.0), (0.0, 10.0), (-10.0, 0.0), (0.0, -10.0)]
    cases = [
        run_case("pf_gate_some_steps_kidnap", rng, 0, 12, 14, c1, 0.5, 0.3, 0.1, 0.1, 0.6, [0.0, 12.0, 0.0, 10.0], thr=0.5,
                 kidnap=(5, 4.0, 2.5)),
        run_case("mcl_fixed_kidnap", rng, 1, 8, 10, ring, 0.4, 0.2, 0.05, 0.1, 0.6, [-8.0, 8.0, -8.0, 8.0], start=(0.0, 0.0, 0.0),
                 kidnap=(4, 3.0, -4.0)),
        run_case("mcl_kld_from_region", rng, 1, 8, 10, ring, 0.4, 0.2, 0.05, 0.1, 0.6, [-2.0, 4.0, -5.0, 1.0], nmax=24, eps=0.5,
                 start=(1.0, -2.0, 0.3), init_region=True, far_at=(3, 4, 5, 6)),
        run_case("mcl_kidnap_s_zero", rng, 1, 8, 10, ring, 0.4, 0.2, 0.05, 0.1, 0.6, [-8.0, 8.0, -8.0, 8.0], start=(0.0, 0.0, 0.0),
                 far_at=(3, 4, 5, 6, 7)),
    ]
    for c in cases:
        inj = [s["injected"] for s in c["steps"]]
        assert any(inj), f"{c['name']}: no step injected"
        print(c["name"], "injected per step", inj, "resampled", [int(s["did_resample"]) for s in c["steps"]])
    path = os.path.join(HERE, "recovery_golden.json")
    with open(path, "w") as f:
        json.dump({"cases": cases}, f, separators=(",", ":"))
    print("wrote recovery_golden.json", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
