#!/usr/bin/env python3
"""Golden vectors of the FastSLAM 2.0 step with UNKNOWN data association (DESIGN §3.5), from a pure-Python restatement.

Run:  python tests/golden/make_assoc_golden.py      -> tests/golden/fs2_assoc_golden.json

The proposal, the pose sample, update_landmark_and_weight, normalise, N_eff and resample are make_golden.py's independent
restatements of fs2.rs (imported, not rewritten); what is stated here is the association rule (search_correspond_landmark_id,
ekf_slam.rs:284-308, evaluated per particle) and the step around it: births in the lowest empty slot, drops when the map is
full.  Python floats are IEEE f64 and math.* is glibc, so tests/host/fs2_assoc_oracle.c built with -DPF_ORACLE_LIBM must
reproduce this file bit for bit (tests/test_fs2_assoc_oracle.py).  The other golden files are not touched.
"""
import json
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import (FP, fs2_compute_proposal, fs2_motion_model, fs2_sample_pose, fs2_update_landmark_and_weight,  # noqa: E402
                         fs_neff, fs_normalize, fs_resample, fs_state, gadd, gmm, gtr, hx, inv2, normalize_angle)

F64_MAX = sys.float_info.max


def assoc_d2(L, pose, z, cfg):
    """y^T S^-1 y with y, S as fs2.rs:258-262 forms them; None when S is singular (try_inverse fails, ekf_slam.rs:293)"""
    dx, dy = L[0] - pose[0], L[1] - pose[1]
    z_pred = [math.sqrt(dx * dx + dy * dy), normalize_angle(math.atan2(dy, dx) - pose[2])]
    y = [[z[0] - z_pred[0]], [normalize_angle(z[1] - z_pred[1])]]
    d2 = dx * dx + dy * dy
    d = math.sqrt(d2)
    h = [[dx / d, dy / d], [-dy / d2, dx / d2]]
    s = gadd(gmm(gmm(h, [[L[2], L[3]], [L[4], L[5]]]), gtr(h)), [[cfg["r00"], 0.0], [0.0, cfg["r11"]]])
    si = inv2(s)
    if si is None:
        return None
    return gmm(gmm(gtr(y), si), y)[0][0]


def associate(p, pose, z, gate, cfg):
    best, bl = F64_MAX, None
    for l, L in enumerate(p.lms):
        if not L[2] < 100.0:
            continue
        q = assoc_d2(L, pose, z, cfg)
        if q is not None and q < best:
            best, bl = q, l
    return bl if bl is not None and best < gate else None


def run_case(name, rng, n, m, T, nth, lm_true, gate=16.0, seeded=0, zero_weights_at=None, no_obs_at=None, dup_at=None):
    cfg = {"dt": 0.1, "max_range": 20.0, "nth": nth, "q00": 0.3, "q11": 0.0305, "r00": 0.5, "r11": 0.0305, "init_weight": 0.01}
    ps = []
    for _ in range(n):
        lms = [[0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0] for _ in range(m)]
        for l in range(min(seeded, m)):                                   # slot l holds a guess of landmark l
            lms[l] = [lm_true[l][0] + rng.normal(), lm_true[l][1] + rng.normal(), 10.0, 0.0, 0.0, 10.0]
        ps.append(FP(cfg["init_weight"], 0.0, 0.0, 0.0, lms))
    pose0, lm0 = fs_state(ps)
    case = {"name": name, "n": n, "m": m, "gate": hx(gate), "cfg": {k: hx(v) for k, v in cfg.items()},
            "init_pose": [hx(r) for r in pose0], "init_lm": [[hx(l) for l in row] for row in lm0], "steps": []}
    xt = [0.0, 0.0, 0.0]
    for t in range(T):
        u = [1.0, 0.1]
        xt = fs2_motion_model(xt, u, cfg["dt"])
        obs = []
        if no_obs_at != t:
            for lx, ly in lm_true:
                dx, dy = lx - xt[0], ly - xt[1]
                d = math.sqrt(dx * dx + dy * dy)
                if d <= cfg["max_range"]:
                    obs.append([d + rng.normal() * math.sqrt(cfg["r00"]),
                                normalize_angle(math.atan2(dy, dx) - xt[2]) + rng.normal() * math.sqrt(cfg["r11"])])
        if dup_at == t and obs:
            obs.append(list(obs[0]))                                      # two observations of one landmark
        z0, z1, z2 = (rng.normal(size=n).tolist() for _ in range(3))
        u01 = float(rng.uniform())
        if zero_weights_at == t:
            for p in ps:
                p.w = 0.0
        counts = [0, 0, 0]
        for i, p in enumerate(ps):
            if obs:
                x_pred = fs2_motion_model([p.x, p.y, p.yaw], u, cfg["dt"])
                l = associate(p, x_pred, obs[0], gate, cfg)
                if l is None:                                             # compute_proposal's uninitialised branch
                    q = FP(p.w, p.x, p.y, p.yaw, [[0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0]])
                    mean, cov = fs2_compute_proposal(q, u, obs[0], 0, cfg)
                else:
                    mean, cov = fs2_compute_proposal(p, u, obs[0], l, cfg)
                sp = fs2_sample_pose(mean, cov, [z0[i], z1[i], z2[i]])
            else:
                un = [u[0] + z0[i] * math.sqrt(cfg["q00"]), u[1] + z1[i] * math.sqrt(cfg["q11"])]
                sp = fs2_motion_model([p.x, p.y, p.yaw], un, cfg["dt"])
            p.x, p.y, p.yaw = sp[0], sp[1], normalize_angle(sp[2])
            for zz in obs:
                l = associate(p, [p.x, p.y, p.yaw], zz, gate, cfg)
                if l is not None:
                    counts[0] += 1
                else:
                    l = next((e for e, L in enumerate(p.lms) if not L[2] < 100.0), None)
                    if l is None:
                        counts[2] += 1
                        continue
                    counts[1] += 1
                p.w *= fs2_update_landmark_and_weight(p, zz, l, cfg)
        fs_normalize(ps)
        neff = fs_neff(ps)
        did = neff < cfg["nth"]
        idxs = []
        if did:
            ps, idxs = fs_resample(ps, u01)
        pose, lm = fs_state(ps)
        case["steps"].append({"u": hx(u), "obs": [hx(o) for o in obs], "z0": hx(z0), "z1": hx(z1), "z2": hx(z2), "u01": hx(u01),
                              "zero_weights": zero_weights_at == t, "neff": hx(neff), "did_resample": bool(did), "indices": idxs,
                              "counts": counts, "pose": [hx(r) for r in pose], "lm": [[hx(l) for l in row] for row in lm]})
    return case


def main():
    rng = np.random.default_rng(20261015)
    lm6 = [(10.0, -2.0), (15.0, 10.0), (3.0, 15.0), (-5.0, 20.0), (-5.0, 5.0), (25.0, 25.0)]
    out = {"cases": [
        run_case("fresh_map_births", rng, n=8, m=8, T=6, nth=8 / 1.5, lm_true=lm6),
        run_case("seeded_and_fresh", rng, n=12, m=6, T=6, nth=12 / 1.5, lm_true=lm6, seeded=3, dup_at=2),
        run_case("full_map_drops", rng, n=6, m=2, T=5, nth=6 / 1.5, lm_true=lm6),
        run_case("gate_inf_no_obs_zero_weights", rng, n=6, m=4, T=5, nth=6 / 1.5, lm_true=lm6[:4], gate=math.inf, no_obs_at=1,
                 zero_weights_at=3),
        run_case("tight_gate", rng, n=10, m=10, T=5, nth=10 / 1.5, lm_true=lm6, gate=0.5, seeded=6),
    ]}
    path = os.path.join(HERE, "fs2_assoc_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, separators=(",", ":"))
    print("wrote fs2_assoc_golden.json", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
