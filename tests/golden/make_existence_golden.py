#!/usr/bin/env python3
"""Golden vectors of the landmark existence counters (DESIGN §3.7) on the FastSLAM 2.0 step with unknown data association.

Run:  python tests/golden/make_existence_golden.py      -> tests/golden/fs2_existence_golden.json

The association is make_assoc_golden.py's, the proposal, the pose sample, update_landmark_and_weight, normalise, N_eff and
resample are make_golden.py's (imported, not rewritten).  What is stated here is the counter: per slot an int tau, cloned with its
particle on resample; a match sets tau += 1, a birth tau = 1, a drop changes nothing; then every initialised slot (cov00 < 100)
that no observation of the step went to and that lies within r of the sampled pose (sqrt(dx*dx + dy*dy) <= r) gets tau -= 1,
and a slot whose tau falls below 0 is removed (reset to create_particles' fresh landmark).  Python floats are IEEE f64 and math.*
is glibc, so tests/host/fs2_exist_oracle.c built with -DPF_ORACLE_LIBM must reproduce this file bit for bit
(tests/test_fs2_existence_oracle.py).
"""
import json
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_assoc_golden import associate  # noqa: E402
from make_golden import (FP, fs2_compute_proposal, fs2_motion_model, fs2_sample_pose, fs2_update_landmark_and_weight,  # noqa: E402
                         fs_neff, fs_normalize, fs_resample, fs_state, hx, normalize_angle)

FRESH = [0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0]


def step_particle(p, tau, u, obs, gate, r, draws, cfg, counts):
    """one particle's unknown-association step with counters; returns the copies it removed"""
    z0, z1, z2 = draws
    if obs:
        x_pred = fs2_motion_model([p.x, p.y, p.yaw], u, cfg["dt"])
        l = associate(p, x_pred, obs[0], gate, cfg)
        if l is None:
            q = FP(p.w, p.x, p.y, p.yaw, [list(FRESH)])
            mean, cov = fs2_compute_proposal(q, u, obs[0], 0, cfg)
        else:
            mean, cov = fs2_compute_proposal(p, u, obs[0], l, cfg)
        sp = fs2_sample_pose(mean, cov, [z0, z1, z2])
    else:
        un = [u[0] + z0 * math.sqrt(cfg["q00"]), u[1] + z1 * math.sqrt(cfg["q11"])]
        sp = fs2_motion_model([p.x, p.y, p.yaw], un, cfg["dt"])
    p.x, p.y, p.yaw = sp[0], sp[1], normalize_angle(sp[2])
    seen = set()
    for zz in obs:
        l = associate(p, [p.x, p.y, p.yaw], zz, gate, cfg)
        if l is not None:
            counts[0] += 1
            tau[l] += 1
        else:
            l = next((e for e, L in enumerate(p.lms) if not L[2] < 100.0), None)
            if l is None:
                counts[2] += 1
                continue
            counts[1] += 1
            tau[l] = 1
        seen.add(l)
        p.w *= fs2_update_landmark_and_weight(p, zz, l, cfg)
    removed = 0
    for l, L in enumerate(p.lms):
        if l in seen or not L[2] < 100.0:
            continue
        dx, dy = L[0] - p.x, L[1] - p.y
        if math.sqrt(dx * dx + dy * dy) <= r:
            tau[l] -= 1
            if tau[l] < 0:
                p.lms[l] = list(FRESH)
                removed += 1
    return removed


def run_case(name, rng, n, m, T, nth, lm_true, r, gate=16.0, init=None, no_obs_at=(), dup_at=None, u=(1.0, 0.1), zero_draws=False):
    """init: (n, m, 6) initial maps (default: fresh); lm_true: the landmarks that produce observations"""
    cfg = {"dt": 0.1, "max_range": 20.0, "nth": nth, "q00": 0.3, "q11": 0.0305, "r00": 0.5, "r11": 0.0305, "init_weight": 0.01}
    ps = [FP(cfg["init_weight"], 0.0, 0.0, 0.0, [list(init[i][l]) if init is not None else list(FRESH) for l in range(m)]) for i in range(n)]
    taus = [[1] * m for _ in range(n)]
    pose0, lm0 = fs_state(ps)
    case = {"name": name, "n": n, "m": m, "gate": hx(gate), "range": hx(r), "cfg": {k: hx(v) for k, v in cfg.items()},
            "init_pose": [hx(v) for v in pose0], "init_lm": [[hx(v) for v in row] for row in lm0], "steps": []}
    xt = [0.0, 0.0, 0.0]
    u = list(u)
    for t in range(T):
        xt = fs2_motion_model(xt, u, cfg["dt"])
        obs = []
        if t not in no_obs_at:
            for lx, ly in lm_true:
                dx, dy = lx - xt[0], ly - xt[1]
                d = math.sqrt(dx * dx + dy * dy)
                if d <= cfg["max_range"]:
                    obs.append([d + rng.normal() * math.sqrt(cfg["r00"]),
                                normalize_angle(math.atan2(dy, dx) - xt[2]) + rng.normal() * math.sqrt(cfg["r11"])])
        if dup_at == t and obs:
            obs.append(list(obs[0]))                                      # two observations of one landmark
        if zero_draws:
            z0, z1, z2 = [0.0] * n, [0.0] * n, [0.0] * n
        else:
            z0, z1, z2 = (rng.normal(size=n).tolist() for _ in range(3))
        u01 = float(rng.uniform())
        counts, removed = [0, 0, 0], 0
        for i, p in enumerate(ps):
            removed += step_particle(p, taus[i], u, obs, gate, r, (z0[i], z1[i], z2[i]), cfg, counts)
        fs_normalize(ps)
        neff = fs_neff(ps)
        did = neff < cfg["nth"]
        idxs = []
        if did:
            ps, idxs = fs_resample(ps, u01)
            taus = [list(taus[j]) for j in idxs]                           # tau is cloned with its particle
        pose, lm = fs_state(ps)
        tau_out = [[taus[i][l] if ps[i].lms[l][2] < 100.0 else 0 for l in range(m)] for i in range(n)]
        case["steps"].append({"u": hx(u), "obs": [hx(o) for o in obs], "z0": hx(z0), "z1": hx(z1), "z2": hx(z2), "u01": hx(u01),
                              "neff": hx(neff), "did_resample": bool(did), "indices": idxs, "counts": counts, "removed": removed,
                              "tau": tau_out, "pose": [hx(v) for v in pose], "lm": [[hx(v) for v in row] for row in lm]})
    return case


def main():
    rng = np.random.default_rng(20261016)
    lm6 = [(10.0, -2.0), (15.0, 10.0), (3.0, 15.0), (-5.0, 20.0), (-5.0, 5.0), (25.0, 25.0)]

    def phantoms(n, m, spots):                                            # slots 0.. hold landmarks that nothing observes
        init = [[list(FRESH) for _ in range(m)] for _ in range(n)]
        for i in range(n):
            for l, (x, y) in enumerate(spots):
                init[i][l] = [x + rng.normal() * 0.1, y + rng.normal() * 0.1, 1.0, 0.0, 0.0, 1.0]
        return init

    def seeded(n, m, k):
        init = [[list(FRESH) for _ in range(m)] for _ in range(n)]
        for i in range(n):
            for l in range(k):
                init[i][l] = [lm6[l][0] + rng.normal(), lm6[l][1] + rng.normal(), 10.0, 0.0, 0.0, 10.0]
        return init

    # the range edge: k = 0, u = 0 and draws 0 keep every pose at exactly (0, 0, 0); d = 5 is decremented, one ulp more is not
    edge = [[[5.0, 0.0, 1.0, 0.0, 0.0, 1.0], [math.nextafter(5.0, math.inf), 0.0, 1.0, 0.0, 0.0, 1.0], [0.0, -5.0, 1.0, 0.0, 0.0, 1.0],
             list(FRESH)] for _ in range(4)]
    assert math.sqrt(edge[0][1][0] ** 2) > 5.0
    out = {"cases": [
        run_case("fresh_map_fills_and_frees", rng, n=6, m=4, T=8, nth=6 / 1.5, lm_true=lm6, r=20.0,
                 init=phantoms(6, 4, [(2.0, 6.0), (6.0, 3.0)])),
        run_case("seeded_map_dup_k0", rng, n=6, m=5, T=6, nth=6 / 1.5, lm_true=lm6, r=8.0, init=seeded(6, 5, 3), dup_at=2,
                 no_obs_at=(4,)),
        run_case("range_edge_k0", rng, n=4, m=4, T=3, nth=0.0, lm_true=[], r=5.0, init=edge, u=(0.0, 0.0), zero_draws=True),
        run_case("range_inf", rng, n=6, m=4, T=5, nth=6 / 1.5, lm_true=lm6[:3], r=math.inf, init=phantoms(6, 4, [(30.0, -30.0)])),
        run_case("full_map_drops_then_births", rng, n=4, m=3, T=5, nth=4 / 1.5, lm_true=lm6, r=20.0,
                 init=phantoms(4, 3, [(1.0, 1.0), (4.0, -3.0), (-2.0, 2.0)]), no_obs_at=(0,)),
    ]}
    path = os.path.join(HERE, "fs2_existence_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, separators=(",", ":"))
    print("wrote fs2_existence_golden.json", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
