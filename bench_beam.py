#!/usr/bin/env python3
"""bench_beam.py — the beam scan model (DESIGN §3.11): what a beam step costs on the GPU, against the likelihood field at the same shape.

    python bench_beam.py --steps 20 --warmup 5 [--runs 2] [--workloads plan_track16,plan_track20,plan_global20,big_track20,...]

bench_scan.py's protocol: W warm-up steps, the L2 flushed before every timed step, one event pair per step, `runs` repeats with the
workloads in alternating order, the median per workload.  MCL at a fixed particle count, ScanScenario's 360-beam scans with max_beams
60.  A workload is <map>_<cloud><log2 n>: map "plan" (the 40 m x 30 m floor plan at 5 cm, 800 x 600 cells) or "big" (the plan tiled to
8192 x 8192); cloud "track" (starts at the truth) or "global" (redrawn uniformly over the map by init_region, outside the timed window,
before every timed step).  Reported per workload:
  beam_us / lfield_us       step time under the beam model and under the likelihood field, in the same call
  beam_noskip_us            the beam step with PFGPU_BEAM_SKIP=0 (the caster steps one cell at a time; one run)
  weight_kernel_us          the beam weight kernel alone (events around it, a pass of its own, no graph)
  set_ms                    set_beam_model (clearance table on the device), host clock around the synchronising call
  probes_per_ray            mean cells read per ray with and without skipping, counted on the host over a sample of the cloud's
                            rays with the device's clearance table
The card's name, power limit and SM clock are on the same JSON line.  Writes nothing into the tree.
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
DEFAULT = "plan_track16,plan_global16,plan_track20,plan_global20,big_track16,big_global16,big_track20,big_global20"


def parse(key):
    m, rest = key.split("_")
    cloud = rest.rstrip("0123456789")
    return m, cloud, 1 << int(rest[len(cloud):])


def make(key, scs, model, skip=True):
    m, _, n = parse(key)
    sc = scs[m]
    g = rr.MonteCarloLocalizer.try_with_initial_state([*sc.truth[0][:3], 1.0], rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.2, 0.1, 0.1),
                                                      seed=42)
    old = os.environ.get("PFGPU_BEAM_SKIP")
    os.environ["PFGPU_BEAM_SKIP"] = "1" if skip else "0"
    try:
        t0 = time.perf_counter()
        if model == "beam":
            g.set_beam_model(sc.obstacles, sc.RES, max_beams=MAX_BEAMS)
        else:
            g.set_likelihood_field(sc.obstacles, sc.RES, max_beams=MAX_BEAMS)
        set_ms = (time.perf_counter() - t0) * 1e3
    finally:
        if old is None:
            os.environ.pop("PFGPU_BEAM_SKIP")
        else:
            os.environ["PFGPU_BEAM_SKIP"] = old
    return g, sc, set_ms


def step(model, g, sc, t):
    args = (sc.controls[t % len(sc.controls)], *sc.scan_args(t % len(sc.controls)))
    (g.try_step_beam_scan if model == "beam" else g.try_step_scan)(*args, want_estimate=False)


def run(key, scs, K, W, model, skip=True, kernel_timer=False):
    g, sc, set_ms = make(key, scs, model, skip)
    glob = parse(key)[1] == "global"
    if kernel_timer:
        g.time_main_kernel(True)
    for t in range(W):
        step(model, g, sc, t)
    g.sync()
    for k in range(K):
        if glob:
            g.init_region(sc.region)
        g.flush_l2()
        g.mark(2 * k)
        step(model, g, sc, W + k)
        g.mark(2 * k + 1)
    g.sync()
    us = sum(g.elapsed_ms(2 * k, 2 * k + 1) for k in range(K)) * 1e3 / K
    st = g.stats()
    kern = st.main_kernel_ms_sum * 1e3 / max(st.main_kernel_count, 1) if kernel_timer else None
    g.close()
    return us, kern, set_ms


def probes(key, scs, W, sample=2048):
    """mean cells read per ray with and without skipping, over `sample` rays of the cloud a timed step weighs (host, numpy: the
    closed form of pf_beam.cuh walked with the device's clearance table)"""
    m, cloud, _ = parse(key)
    sc = scs[m]
    g, _, _ = make(key, scs, "beam")
    for t in range(W):
        step("beam", g, sc, t)
    if cloud == "global":
        g.init_region(sc.region)
    clr = g.beam_model().astype(np.int64)
    p = g.get_particles()
    g.close()
    rng = np.random.default_rng(1)
    p = p[rng.integers(0, len(p), sample // MAX_BEAMS + 1)]
    r, amin, ainc = sc.scan_args(W % len(sc.controls))
    s = max(1, (len(r) - 1) // (MAX_BEAMS - 1))
    ang = (p[:, 2:3] + amin) + (np.arange(0, len(r), s) * ainc)[None, :]
    x, y, ang = np.repeat(p[:, 0], ang.shape[1]), np.repeat(p[:, 1], ang.shape[1]), ang.ravel()
    Wc, Hc = clr.shape
    cell = lambda v, half: np.floor(v / sc.RES + half).astype(np.int64)
    ix0, iy0 = cell(x, Wc / 2.0), cell(y, Hc / 2.0)
    ix1, iy1 = cell(x + 30.0 * np.cos(ang), Wc / 2.0), cell(y + 30.0 * np.sin(ang), Hc / 2.0)
    dx, dy = ix1 - ix0, iy1 - iy0
    xm = np.abs(dx) >= np.abs(dy)
    dM, dm = np.where(xm, np.abs(dx), np.abs(dy)), np.where(xm, np.abs(dy), np.abs(dx))
    sx, sy = np.where(ix0 < ix1, 1, -1), np.where(iy0 < iy1, 1, -1)
    inside0 = (ix0 >= 0) & (ix0 < Wc) & (iy0 >= 0) & (iy0 < Hc)
    out = []
    for skip in (True, False):
        i = np.zeros_like(dM)
        live = inside0.copy()
        count = np.zeros_like(dM)
        while live.any():
            mi = np.where(dm == 0, 0, (2 * i * dm + dM - 1) // np.maximum(2 * dM, 1))
            cx, cy = ix0 + sx * np.where(xm, i, mi), iy0 + sy * np.where(xm, mi, i)
            ok = live & (cx >= 0) & (cx < Wc) & (cy >= 0) & (cy < Hc)
            c = np.where(ok, clr[np.clip(cx, 0, Wc - 1), np.clip(cy, 0, Hc - 1)], 0)
            count += live
            live = ok & (c > 0)
            i = np.where(live, i + (c if skip else 1), i)
            live &= i <= dM
        out.append(float(count.mean()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--workloads", default=DEFAULT)
    a = ap.parse_args()
    keys = [k for k in a.workloads.split(",") if k]
    scs = {"plan": scenarios.ScanScenario(steps=60)}
    if any(k.startswith("big") for k in keys):
        scs["big"] = scenarios.ScanScenario(steps=60, cells=8192)
    sampler = bench.ClockSampler(0)
    times = {(k, mdl): [] for k in keys for mdl in ("beam", "lfield")}
    for r in range(a.runs):
        order = [(k, mdl) for k in keys for mdl in ("beam", "lfield")]
        for k, mdl in (order if r % 2 == 0 else order[::-1]):
            times[(k, mdl)].append(run(k, scs, a.steps, a.warmup, mdl))
    out = {}
    for k in keys:
        _, kern, _ = run(k, scs, a.steps, a.warmup, "beam", kernel_timer=True)
        noskip, _, _ = run(k, scs, a.steps, a.warmup, "beam", skip=False)
        pr = probes(k, scs, a.warmup)
        out[k] = {"particles": parse(k)[2], "map_cells": list(scs[parse(k)[0]].obstacles.shape),
                  "beam_us": statistics.median(u for u, _, _ in times[(k, "beam")]),
                  "lfield_us": statistics.median(u for u, _, _ in times[(k, "lfield")]),
                  "beam_noskip_us": noskip, "weight_kernel_us": kern,
                  "set_ms": statistics.median(s for _, _, s in times[(k, "beam")]),
                  "probes_per_ray": {"skip": pr[0], "noskip": pr[1]}}
        print(json.dumps({"workload": k, **out[k]}), file=sys.stderr, flush=True)
    print(json.dumps({"metric": "beam scan step", "steps": a.steps, "warmup": a.warmup, "runs": a.runs, "max_beams": MAX_BEAMS,
                      "workloads": out, "gpu": bench.gpu_info(0), "clocks": sampler.stop()}))


if __name__ == "__main__":
    main()
