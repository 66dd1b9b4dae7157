#!/usr/bin/env python3
"""bench_gslam.py — grid-based FastSLAM on the device (DESIGN §3.16): what one step of laser SLAM with a grid per particle costs.

    python bench_gslam.py [--runs 3] [--sizes 256,1024,4096] [--steps 40]

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


def make(sc, n, seed=7):
    W, H = sc.obstacles.shape
    return rr.GridFastSlam(rr.GridFastSlamConfig(rr.OccupancyGridConfig(resolution=sc.RES, width=W, height=H), n_particles=n),
                           start_pose=sc.start, seed=seed)


def step(sc, g, t):
    prev, cur = sc.odom_pair(t)
    g.step(prev, cur, sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)


def timed_run(sc, n, steps, flusher):
    g = make(sc, n)
    us, events, copies = [], [], []
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
    g.close()
    return statistics.median(us), float(np.mean(events)), (float(np.mean(copies)) if copies else 0.0), len(copies)


def kind_of(name):
    if "gs_move_weigh" in name:
        return "move_weigh"
    if "gs_fuse" in name:
        return "fuse"
    if "gs_copy" in name:
        return "copy"
    if "pf_l2_read" in name or "Memset" in name or "Memcpy" in name:
        return "other"
    return "sums_gate_comb"


def profile(sc, n, steps):
    from torch.profiler import ProfilerActivity, profile as prof
    g = make(sc, n)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--sizes", default="256,1024,4096")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--cpu-steps", type=int, default=12)
    a = ap.parse_args()
    sc = scenarios.OdomScenario()
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
