#!/usr/bin/env python3
"""bench_scan.py — the likelihood-field scan model (DESIGN §3.9): what a scan step costs on the GPU.

    python bench_scan.py --steps K --warmup W [--runs 4] [--workloads plan_track,plan_global,big_track,big_global,fused16,landmark20]

bench.py's PF / MCL protocol: W warm-up steps, the L2 flushed before every timed step, one event pair per step, `runs` repeats with
the workloads in alternating order, the median per workload.  All MCL at a fixed particle count, ScanScenario's 360-beam scans with
max_beams 60 (60 used beams when every candidate returns):
  plan_track / plan_global   2^20 particles on the 40 m x 30 m floor plan at 5 cm (800 x 600 cells: a 3.8 MB table, in L2)
  big_track / big_global     the same on an 8192 x 8192 map (the plan tiled; a 512 MB table, in HBM)
  fused16                    2^16 particles tracking on the plan (the fused step)
  landmark20                 config 2's landmark step (360 landmarks) at 2^20, for contrast
"track" starts at the truth; "global" redraws the cloud uniformly over the map (init_region, outside the timed window) before every
timed step, so each timed step weighs a cloud spread over the whole map.  Reported per workload: step time, weight-kernel time
(a separate run with per-kernel events, no graph), particle-beam evaluations per second over the weight kernel, algorithmic bytes
per step (8 B per beam gather + the 32 B pose record per particle) and the set time (distance field + table, host clock around the
synchronising call).  The card's name, power limit and SM clock are on the same JSON line.  Writes nothing into the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402
import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import scenarios  # noqa: E402

MAX_BEAMS = 60


def used_beams(r, max_range=30.0):
    s = max(1, (len(r) - 1) // (MAX_BEAMS - 1))
    c = np.asarray(r)[::s]
    return int(np.count_nonzero((c > 0.0) & np.isfinite(c) & (c < max_range)))


def make(key, scs):
    n = 1 << 16 if key == "fused16" else 1 << 20
    cfg = rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.2, 0.1, 0.1)
    if key == "landmark20":
        sc = scs["c2"]
        return rr.MonteCarloLocalizer.try_with_initial_state(sc.init, rr.MonteCarloLocalizationConfig(*scenarios.KidnapScenario.config(n))), sc, n, None
    sc = scs["big" if key.startswith("big") else "plan"]
    g = rr.MonteCarloLocalizer.try_with_initial_state([*sc.truth[0][:3], 1.0], cfg, seed=42)
    t0 = time.perf_counter()
    g.set_likelihood_field(sc.obstacles, sc.RES, max_beams=MAX_BEAMS)
    return g, sc, n, (time.perf_counter() - t0) * 1e3


def step(key, g, sc, t):
    if key == "landmark20":
        g.try_step(sc.controls[t], sc.obs[t], want_estimate=False)
    else:
        g.try_step_scan(sc.controls[t % len(sc.controls)], *sc.scan_args(t % len(sc.controls)), want_estimate=False)


def run(key, scs, K, W, kernel_timer=False):
    g, sc, n, set_ms = make(key, scs)
    glob = key.endswith("global")
    if kernel_timer:
        g.time_main_kernel(True)
    for t in range(W):
        step(key, g, sc, t)
    g.sync()
    for k in range(K):
        if glob:
            g.init_region(sc.region)
        g.flush_l2()
        g.mark(2 * k)
        step(key, g, sc, W + k)
        g.mark(2 * k + 1)
    g.sync()
    us = sum(g.elapsed_ms(2 * k, 2 * k + 1) for k in range(K)) * 1e3 / K
    st = g.stats()
    kern = st.main_kernel_ms_sum * 1e3 / max(st.main_kernel_count, 1) if kernel_timer else None
    g.close()
    return us, kern, n, set_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=4)
    ap.add_argument("--workloads", default="plan_track,plan_global,big_track,big_global,fused16,landmark20")
    a = ap.parse_args()
    keys = [k for k in a.workloads.split(",") if k]
    steps = a.warmup + a.steps
    scs = {"plan": scenarios.ScanScenario(steps=60), "c2": scenarios.PfScenario("c2", steps=steps)}
    if any(k.startswith("big") for k in keys):
        scs["big"] = scenarios.ScanScenario(steps=60, cells=8192)
    sampler = bench.ClockSampler(0)
    times = {k: [] for k in keys}
    for r in range(a.runs):
        for k in (keys if r % 2 == 0 else keys[::-1]):
            times[k].append(run(k, scs, a.steps, a.warmup))
    out = {}
    for k in keys:
        us = statistics.median(u for u, _, _, _ in times[k])
        _, kern, n, _ = run(k, scs, a.steps, a.warmup, kernel_timer=True)
        res = {"particles": n, "us_per_step": us, "weight_kernel_us": kern}
        if k != "landmark20":
            sc = scs["big" if k.startswith("big") else "plan"]
            beams = float(np.mean([used_beams(sc.scans[(a.warmup + j) % len(sc.scans)]) for j in range(a.steps)]))
            res.update({"map_cells": list(sc.obstacles.shape), "used_beams_mean": beams,
                        "beam_evals_per_s": n * beams / (kern * 1e-6) if kern else None,
                        "algorithmic_bytes_per_step": n * (8.0 * beams + 32.0),
                        "set_ms": statistics.median(s for _, _, _, s in times[k])})
        out[k] = res
    print(json.dumps({"metric": "likelihood-field scan step", "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "max_beams": MAX_BEAMS,
                      "workloads": out, "gpu": bench.gpu_info(0), "clocks": sampler.stop()}))


if __name__ == "__main__":
    main()
