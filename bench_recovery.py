#!/usr/bin/env python3
"""bench_recovery.py — augmented MCL (DESIGN §3.8): what random-particle injection costs per step, and what it buys.

    python bench_recovery.py --steps K --warmup W [--runs 4] [--configs mcl20,pf16,pf18] [--sizes 14,16,18,20]     # one JSON line

Cost: bench.py's PF / MCL protocol (L2 flushed before every timed step, one event pair per step, W warm-up steps), recovery off /
on (alpha_slow 0.001, alpha_fast 0.1) in `runs` alternating runs, median per setting: us and kernel launches per step.  mcl20 =
config 2 (MCL, 2^20 particles, 360 beams); pf16 / pf18 = the config-5 points (PF, C1 model, threshold 1.0).  These runs track
(p = 0), so "on" is the cost of the machinery.  Behaviour: KidnapScenario (30 steps of tracking, a 15 m kidnap, 60 more steps) at
2^14 .. 2^20 particles, alpha_slow 0.01, alpha_fast 0.2: steps after the kidnap until the estimate is within 1 m (null: never), off
and on, and particles injected per step; global localisation from init_region: steps until within 1 m.  The card's name, power
limit and SM clock are on the same line.  Writes nothing into the tree.
"""
import argparse
import json
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


def cost_run(key, on, K, W):
    if key == "mcl20":
        sc = scenarios.PfScenario("c2", steps=W + K)
        g = rr.MonteCarloLocalizer.try_with_initial_state(sc.init, rr.MonteCarloLocalizationConfig(*scenarios.KidnapScenario.config(1 << 20)), seed=42)
        box = scenarios.KidnapScenario.REGION
    else:
        sc = scenarios.PfScenario("c1", steps=W + K)
        g = rr.ParticleFilterLocalizer.try_with_initial_state(sc.init, rr.ParticleFilterConfig(1 << int(key[2:]), 1.0, 0.25), seed=42)
        box = (-5.0, 15.0, -5.0, 15.0)
    if on:
        g.enable_recovery(0.001, 0.1, box)
    obs, ctl = [np.ascontiguousarray(o) for o in sc.obs], [np.asarray(c, dtype=np.float64) for c in sc.controls]
    for t in range(W):
        g.try_step(ctl[t], obs[t], want_estimate=False)
    g.sync()
    s0 = g.stats().kernel_launches
    for k in range(K):
        g.flush_l2()
        g.mark(2 * k)
        g.try_step(ctl[W + k], obs[W + k], want_estimate=False)
        g.mark(2 * k + 1)
    g.sync()
    us = sum(g.elapsed_ms(2 * k, 2 * k + 1) for k in range(K)) * 1e3 / K
    return us, (g.stats().kernel_launches - s0) / K


def kidnap(n, on):
    sc = scenarios.KidnapScenario()
    g = rr.MonteCarloLocalizer.try_with_initial_state(sc.init, rr.MonteCarloLocalizationConfig(*sc.config(n)), seed=3)
    if on:
        g.enable_recovery(0.01, 0.2, sc.REGION)
    first, inj = None, []
    for k in range(len(sc.controls)):
        err = sc.error(k, g.try_step(sc.controls[k], sc.obs[k]))
        if k >= sc.before:
            inj.append(g.recovery_state()[3])
            first = first if first is not None or err >= 1.0 else k - sc.before + 1
    return first, float(np.mean(inj))


def global_loc(n):
    sc = scenarios.KidnapScenario(before=0, after=30)
    g = rr.MonteCarloLocalizer.try_with_region(sc.REGION, rr.MonteCarloLocalizationConfig(*sc.config(n)), seed=5)
    g.enable_recovery(0.01, 0.2, sc.REGION)
    return next((k + 1 for k in range(len(sc.controls)) if sc.error(k, g.try_step(sc.controls[k], sc.obs[k])) < 1.0), None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--runs", type=int, default=4)
    ap.add_argument("--configs", default="mcl20,pf16,pf18")
    ap.add_argument("--sizes", default="14,16,18,20")
    a = ap.parse_args()
    sampler = bench.ClockSampler(0)
    cost = {}
    for key in filter(None, a.configs.split(",")):
        res = {False: [], True: []}
        for r in range(a.runs):
            for on in ((False, True) if r % 2 == 0 else (True, False)):
                res[on].append(cost_run(key, on, a.steps, a.warmup))
        us = {on: statistics.median(u for u, _ in res[on]) for on in res}
        cost[key] = {"off_us_per_step": us[False], "on_us_per_step": us[True], "overhead_pct": (us[True] / us[False] - 1.0) * 100.0,
                     "off_launches_per_step": res[False][0][1], "on_launches_per_step": res[True][0][1]}
    behaviour = {}
    for e in (int(s) for s in filter(None, a.sizes.split(","))):
        (off, _), (on, inj) = kidnap(1 << e, False), kidnap(1 << e, True)
        behaviour[f"2^{e}"] = {"kidnap_steps_to_1m_off": off, "kidnap_steps_to_1m_on": on, "injected_per_step": inj,
                               "global_steps_to_1m": global_loc(1 << e)}
    print(json.dumps({"metric": "augmented MCL cost and recovery", "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "cost": cost,
                      "behaviour": behaviour, "gpu": bench.gpu_info(0), "clocks": sampler.stop()}))


if __name__ == "__main__":
    main()
