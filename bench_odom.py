#!/usr/bin/env python3
"""bench_odom.py — the odometry motion model (DESIGN §3.14): what an odometry step costs against its velocity twin, and what it does
for tracking.

    python bench_odom.py --steps K --warmup W [--runs 4]

bench_scan.py's protocol: W warm-up steps, the L2 flushed before every timed step, one event pair per step, `runs` repeats with the
two motion models alternating within each workload (velocity, odometry, velocity, ...), the median per model.  Workloads:
  pf16 / pf18      ParticleFilterLocalizer at 2^16 / 2^18 with config 1's landmark world (PfScenario c1), the PF gate
  mcl20            MonteCarloLocalizer at 2^20 tracking on OdomScenario's floor plan under the likelihood field (60 beams)
The velocity twin steps with OdomScenario's controls (the (v, yaw_rate) that reproduces each odometry step over dt); the odometry
steps take the odometry pairs.  Also: predict-only kernel time at 2^20 (events around K predicts, no weight pass), and on
OdomScenario at 2^16 under the likelihood field from the start pose, the worst position / heading error of each model per phase and
the cloud's spread (sqrt of the x and y variances' sum) at the start and end of the stop.  The card's name, power limit and SM clock
are on the same JSON line.  Writes nothing into the tree.
"""
import argparse
import json
import math
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402
import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import scenarios  # noqa: E402


def make(key, sc, pf):
    n = {"pf16": 1 << 16, "pf18": 1 << 18, "mcl20": 1 << 20}[key]
    if key.startswith("pf"):
        g = rr.ParticleFilterLocalizer.try_with_initial_state(pf.init, rr.ParticleFilterConfig(n, 0.5, 0.25, 0.2, 0.1, 0.1), seed=42)
    else:
        g = rr.MonteCarloLocalizer.try_with_initial_state([*sc.start, 0.0], rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.2, 0.1, 0.1),
                                                          seed=42)
        g.set_likelihood_field(sc.obstacles, sc.RES)
    return g


def step(key, g, sc, pf, t, odom):
    t = t % sc.steps
    if key.startswith("pf"):
        obs = pf.obs[t % len(pf.obs)]
        if odom:
            g.try_step_odometry(*sc.odom_pair(t), obs, want_estimate=False)
        else:
            g.try_step(sc.controls[t], obs, want_estimate=False)
    elif odom:
        g.try_step_scan_odometry(*sc.odom_pair(t), *sc.scan_args(t), want_estimate=False)
    else:
        g.try_step_scan(sc.controls[t], *sc.scan_args(t), want_estimate=False)


def time_steps(key, g, sc, pf, K, W, odom):
    for t in range(W):
        step(key, g, sc, pf, t, odom)
    g.sync()
    ms = []
    for t in range(K):
        g.flush_l2()
        g.mark(0)
        step(key, g, sc, pf, W + t, odom)
        g.mark(1)
        ms.append(g.elapsed_ms(0, 1))
    return statistics.median(ms)


def predict_ms(sc, K, odom):
    n = 1 << 20
    g = rr.MonteCarloLocalizer.try_with_initial_state([*sc.start, 0.0], rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.2, 0.1, 0.1),
                                                      seed=42)
    for t in range(5):
        g.try_predict_with_odometry(*sc.odom_pair(t)) if odom else g.try_predict_with_control(sc.controls[t])
    g.sync()
    g.mark(0)
    for t in range(K):
        g.try_predict_with_odometry(*sc.odom_pair(t % sc.steps)) if odom else g.try_predict_with_control(sc.controls[t % sc.steps])
    g.mark(1)
    return g.elapsed_ms(0, 1) / K


def tracking(sc, odom):
    n = 1 << 16
    g = rr.MonteCarloLocalizer.try_with_initial_state([*sc.start, 0.0], rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.2, 0.1, 0.1),
                                                      seed=5)
    g.set_likelihood_field(sc.obstacles, sc.RES)
    err, spread = [], []
    for t in range(sc.steps):
        e = g.try_step_scan_odometry(*sc.odom_pair(t), *sc.scan_args(t)) if odom else g.try_step_scan(sc.controls[t], *sc.scan_args(t))
        err.append(sc.error(t, e))
        c = g.calc_covariance()
        spread.append(math.sqrt(max(c[0, 0] + c[1, 1], 0.0)))
    err = np.array(err)
    a, b = sc.phases["stop"]
    return {"max_error_m": {k: float(err[s:e, 0].max()) for k, (s, e) in sc.phases.items()},
            "max_heading_error_rad": {k: float(err[s:e, 1].max()) for k, (s, e) in sc.phases.items()},
            "stop_spread_m": [spread[a], spread[b - 1]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--runs", type=int, default=4)
    a = ap.parse_args()
    sc, pf = scenarios.OdomScenario(), scenarios.PfScenario("c1", steps=60)
    out = {"bench": "odom", "gpu": bench.gpu_info(0), "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "step_ms": {}}
    for key in ("pf16", "pf18", "mcl20"):
        runs = {False: [], True: []}
        for r in range(a.runs):
            for odom in ((False, True) if r % 2 == 0 else (True, False)):
                runs[odom].append(time_steps(key, make(key, sc, pf), sc, pf, a.steps, a.warmup, odom))
        out["step_ms"][key] = {"velocity": statistics.median(runs[False]), "odometry": statistics.median(runs[True])}
    out["predict_ms_2^20"] = {"velocity": predict_ms(sc, 4 * a.steps, False), "odometry": predict_ms(sc, 4 * a.steps, True)}
    out["tracking_2^16"] = {"velocity": tracking(sc, False), "odometry": tracking(sc, True)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
