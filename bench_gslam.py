#!/usr/bin/env python3
"""bench_gslam.py — grid-based FastSLAM on the device (DESIGN §3.16): what one step of laser SLAM with a grid per particle costs.

    python bench_gslam.py [--runs 3] [--sizes 256,1024,4096] [--steps 40]
    python bench_gslam.py --proposal [--runs 3] [--sizes 32,128,1024] [--steps 40]

Workload: OdomScenario (82 steps of 360-beam scans and wheel odometry in the 40 m x 30 m floor plan), every particle's grid 800 x 600
at 5 cm (3.84 MB), N = 2^8, 2^10 and 2^12 particles, the default model (R = 1, 60 beams, nth = N / 2).  Per N and run:
  step_us         the median over the timed steps of one step's time: host clock around pfgpu_gs_step plus a synchronise, the L2
                  flushed before each (the first 5 steps are warm-up)
  events          fuse cell updates per step (mean), and cell updates per second of the fuse kernel
  copies          grids copied per resample (mean), the bytes written, and (read + written bytes) / copy time, against 3.35 TB/s (the
                  H100 SXM data sheet's HBM3 bandwidth)
  split_ms        per-kernel device time of one pass over the steps from torch.profiler, in a pass of its own: move + weigh, sums +
                  gate + comb (the exact-sum pipeline, normalisation, search, plan, CUB scans), copy, fuse
  cpu_oracle      tests/host/gs_oracle.c built with glibc libm (compiled into a temporary directory), one host thread, N = 64, at
                  the same grid: ms per step
With --proposal (DESIGN §3.17) the same workload runs with the scan-matched proposal on (the default GridFastSlamProposal) and off,
alternated within each run, at N = 32, 128 and 1024 by default; per N and arm: step_us, resamples and grids copied per step, the
share of particles that took the proposal, and split_ms_per_step with the proposal kernel as "propose".
Runs alternate their order; medians are reported.  The card's name, power limit and SM clock are on the same JSON line.  Writes
nothing into the tree.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch  # noqa: F401  (torch.profiler; loaded before libpfgpu.so so that torch's NCCL is the one resolved)

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402
import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import scenarios  # noqa: E402

HBM_TBS = 3.35
WARM = 5


def make(sc, n, seed=7, prop=False):
    W, H = sc.obstacles.shape
    g = rr.GridFastSlam(rr.GridFastSlamConfig(rr.OccupancyGridConfig(resolution=sc.RES, width=W, height=H), n_particles=n),
                        start_pose=sc.start, seed=seed)
    if prop:
        g.set_proposal(rr.GridFastSlamProposal())
    return g


def step(sc, g, t):
    prev, cur = sc.odom_pair(t)
    g.step(prev, cur, sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)


def timed_run(sc, n, steps, flusher, prop=False):
    g = make(sc, n, prop=prop)
    us, events, copies, took = [], [], [], []
    for t in range(steps):
        flusher.flush_l2()
        flusher.sync()
        g.sync()
        t0 = time.perf_counter()
        step(sc, g, t)
        g.sync()
        dt = (time.perf_counter() - t0) * 1e6
        s = g.stats()
        if t >= WARM:
            us.append(dt)
            events.append(s.events)
            if s.resampled:
                copies.append(s.copies)
            if prop:
                took.append(float(np.mean(g.last_proposal().took)))
    g.close()
    r = statistics.median(us), float(np.mean(events)), (float(np.mean(copies)) if copies else 0.0), len(copies)
    return r + ((float(np.mean(took)), float(np.sum(copies)) / len(us)) if prop else ())


def kind_of(name):
    if "gs_move_weigh" in name:
        return "move_weigh"
    if "gs_propose" in name:
        return "propose"
    if "gs_fuse" in name:
        return "fuse"
    if "gs_copy" in name:
        return "copy"
    if "pf_l2_read" in name or "Memset" in name or "Memcpy" in name:
        return "other"
    return "sums_gate_comb"


def profile(sc, n, steps, prop=False):
    from torch.profiler import ProfilerActivity, profile as prof
    g = make(sc, n, prop=prop)
    for t in range(WARM):
        step(sc, g, t)
    g.sync()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        for t in range(WARM, steps):
            step(sc, g, t)
        g.sync()
    g.close()
    split = {}
    for e in p.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        k = kind_of(e.key)
        split[k] = split.get(k, 0.0) + t / 1e3 / (steps - WARM)
    return {k: round(v, 4) for k, v in sorted(split.items())}


def cpu_oracle(sc, steps, n=64):
    tmp = tempfile.mkdtemp()
    lib = os.path.join(tmp, "libgs_oracle_libm.so")
    subprocess.run(["gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-DPF_ORACLE_LIBM", "-shared", "-o",
                    lib, os.path.join(ROOT, "tests", "host", "gs_oracle.c"), "-lm"], check=True)
    L = C.CDLL(lib)
    dp, sz = C.POINTER(C.c_double), C.c_size_t
    L.orc_gs_new.argtypes, L.orc_gs_new.restype = [dp, sz, sz, dp, sz, C.c_uint64, dp], C.c_void_p
    L.orc_gs_step.argtypes = [C.c_void_p, dp, dp, dp, sz, C.c_double, C.c_double, dp, dp]
    L.orc_gs_free.argtypes = [C.c_void_p]
    W, H = sc.obstacles.shape

    def p(a):
        return np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(dp)
    cfg, model, start = np.array([sc.RES, 0.0, 0.85, -0.4, 5.0, -5.0]), np.array([0.95, 0.05, 30.0, 60, 1, n / 2.0]), np.array(sc.start)
    h = L.orc_gs_new(p(cfg), W, H, p(model), n, 7, p(start))
    alpha = np.full(4, 0.2)
    ms = []
    for t in range(steps):
        o = np.array(list(sc.odom[t]) + list(sc.odom[t + 1]))
        r = np.ascontiguousarray(sc.scans[t])
        t0 = time.perf_counter()
        L.orc_gs_step(h, p(o), p(alpha), r.ctypes.data_as(dp), r.size, sc.ANGLE_MIN, sc.ANGLE_INC, None, None)
        ms.append((time.perf_counter() - t0) * 1e3)
    L.orc_gs_free(h)
    return statistics.median(ms[WARM:])


def proposal_arm(sc, sizes, runs, steps):
    flusher = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(1024, 1024), seed=1)
    sampler = bench.ClockSampler(0)
    res = {(n, p): [] for n in sizes for p in (True, False)}
    for r in range(runs):
        for n in (sizes if r % 2 == 0 else sizes[::-1]):
            for p in ((True, False) if r % 2 == 0 else (False, True)):
                res[(n, p)].append(timed_run(sc, n, steps, flusher, prop=p))
    clocks = sampler.stop()
    out = {}
    for n in sizes:
        for p in (True, False):
            x = res[(n, p)]
            arm = {"step_us": statistics.median(v[0] for v in x), "step_us_runs": [round(v[0], 1) for v in x],
                   "resamples_per_step": x[0][3] / (steps - WARM), "copies_per_resample": x[0][2],
                   "split_ms_per_step": profile(sc, n, steps, prop=p)}
            if p:
                arm["copies_per_step"], arm["took_share"] = x[0][5], x[0][4]
            else:
                arm["copies_per_step"] = x[0][2] * x[0][3] / (steps - WARM)
            out[f"{n}_{'proposal' if p else 'plain'}"] = arm
    W, H = sc.obstacles.shape
    print(json.dumps({"metric": "grid FastSLAM proposal", "runs": runs, "steps": steps, "grid": [W, H], "results": out,
                      "gpu": bench.gpu_info(0), "clocks": clocks}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--sizes", default=None)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--cpu-steps", type=int, default=12)
    ap.add_argument("--proposal", action="store_true")
    a = ap.parse_args()
    sc = scenarios.OdomScenario()
    if a.proposal:
        proposal_arm(sc, [int(s) for s in (a.sizes or "32,128,1024").split(",")], a.runs, min(a.steps, sc.steps))
        return
    a.sizes = a.sizes or "256,1024,4096"
    steps = min(a.steps, sc.steps)
    sizes = [int(s) for s in a.sizes.split(",")]
    flusher = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(1024, 1024), seed=1)
    sampler = bench.ClockSampler(0)
    res = {n: [] for n in sizes}
    for r in range(a.runs):
        for n in (sizes if r % 2 == 0 else sizes[::-1]):
            res[n].append(timed_run(sc, n, steps, flusher))
    clocks = sampler.stop()
    W, H = sc.obstacles.shape
    grid_bytes = W * H * 8
    out = {}
    for n in sizes:
        us = statistics.median(x[0] for x in res[n])
        ev, cp, nres = res[n][0][1], res[n][0][2], res[n][0][3]
        split = profile(sc, n, steps)
        fuse_ms = split.get("fuse", 0.0)
        copy_ms = split.get("copy", 0.0) * (steps - WARM) / max(1, nres)       # per resample
        out[str(n)] = {"step_us": us, "step_us_runs": [round(x[0], 1) for x in res[n]], "events_per_step": ev,
                       "fuse_cell_updates_per_s": ev / (fuse_ms * 1e-3) if fuse_ms else None, "resamples": nres,
                       "copies_per_resample": cp, "bytes_per_resample": cp * grid_bytes,
                       "copy_tb_per_s": (cp * grid_bytes * 2 / (copy_ms * 1e-3) / 1e12) if copy_ms and cp else None,
                       "split_ms_per_step": split}
    out["cpu_oracle_n64_ms_per_step"] = cpu_oracle(sc, a.cpu_steps)
    print(json.dumps({"metric": "grid FastSLAM", "runs": a.runs, "steps": steps, "grid": [W, H], "results": out, "hbm_tb_s_datasheet": HBM_TBS,
                      "gpu": bench.gpu_info(0), "clocks": clocks}))


if __name__ == "__main__":
    main()
