#!/usr/bin/env python3
"""bench_ogm.py — occupancy grid mapping on the device (DESIGN §3.12): what fusing scans into the log-odds grid costs, and what
handing the grid to the PF / MCL scan models costs against the host round trip.

    python bench_ogm.py [--runs 5] [--scans 600]

Workloads (ScanScenario's 360-beam scans from its truth poses; the 600-scan trajectory is its 60 scans ten times over):
  live_plan        one scan per call on the 800 x 600 floor plan at 5 cm: call time (host clock around the synchronising call,
                   the L2 flushed before each), median over 60 calls per run
  traj_plan        all scans in one call on the plan, and traj_big on the plan tiled to 8192 x 8192: call time, cell updates per
                   second, chunks, the longest per-cell run; kernel split from torch.profiler in a pass of its own
  cpu_oracle       tests/host/ogm_oracle.c built with glibc libm (compiled into a temporary directory), one host thread, traj_plan's
                   batch: the sequential reference arm
  hand_off         set_beam_model_from_grid / set_likelihood_field_from_grid, against grid download + obstacles_from_log_odds +
                   set_beam_model / set_likelihood_field from the host mask, on the mapped plan
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


def grid_map(sc, cells=0):
    W, H = sc.obstacles.shape if not cells else (cells, cells)
    return rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=sc.RES, width=W, height=H))


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def live(sc, flusher):
    g = grid_map(sc)
    for t in range(5):                                   # warm-up (the workspace is allocated by the first update)
        g.update_with_scan(*sc.truth[t], sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)
    us = []
    for t in range(len(sc.scans)):
        flusher.flush_l2()
        flusher.sync()
        us.append(timed(lambda: g.update_with_scan(*sc.truth[t], sc.scans[t], sc.ANGLE_MIN, sc.ANGLE_INC)) * 1e3)
    g.close()
    return statistics.median(us)


def traj(sc, poses, scans, flusher, cells=0):
    g = grid_map(sc, cells)
    g.update_with_scans(poses[:60], scans[:60], sc.ANGLE_MIN, sc.ANGLE_INC)       # warm-up
    flusher.flush_l2()
    flusher.sync()
    ms = timed(lambda: g.update_with_scans(poses, scans, sc.ANGLE_MIN, sc.ANGLE_INC))
    st = g.stats()
    g.close()
    return ms, st


def profile(sc, poses, scans, cells, outdir):
    """per-kernel device time of one trajectory call (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile as prof
    g = grid_map(sc, cells)
    g.update_with_scans(poses[:60], scans[:60], sc.ANGLE_MIN, sc.ANGLE_INC)
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        g.update_with_scans(poses, scans, sc.ANGLE_MIN, sc.ANGLE_INC)
        torch.cuda.synchronize()
    g.close()
    split = {}
    for e in p.key_averages():
        name = e.key
        kind = next((k for k in ("count", "chunk", "emit", "fold", "mask") if f"pf_ogm_{k}_kernel" in name), None)
        if kind is None:
            kind = "sort" if "Radix" in name or "Onesweep" in name or "Histogram" in name else ("scan" if "Scan" in name else None)
        if kind is None:
            kind = "copy" if "Memcpy" in name or "Memset" in name else "other"
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        split[kind] = split.get(kind, 0.0) + t / 1e3
    if outdir:
        os.makedirs(outdir, exist_ok=True)
        p.export_chrome_trace(os.path.join(outdir, f"ogm_traj_{cells or 'plan'}.pt.trace.json"))
    return {k: round(v, 3) for k, v in sorted(split.items())}


def cpu_oracle(sc, poses, scans):
    tmp = tempfile.mkdtemp()
    lib = os.path.join(tmp, "libogm_oracle_libm.so")
    subprocess.run(["gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-DPF_ORACLE_LIBM", "-shared", "-o",
                    lib, os.path.join(ROOT, "tests", "host", "ogm_oracle.c"), "-lm"], check=True)
    L = C.CDLL(lib)
    dp = C.POINTER(C.c_double)
    L.orc_ogm_update_scans.argtypes = [dp, dp, C.c_size_t, C.c_size_t, dp, C.c_size_t, dp, C.c_size_t, C.c_double, C.c_double]
    W, H = sc.obstacles.shape
    grid = np.zeros((W, H))
    cfg = np.array([sc.RES, 0.0, 0.85, -0.4, 5.0, -5.0])
    p, r = np.ascontiguousarray(poses), np.ascontiguousarray(scans)
    ms = timed(lambda: L.orc_ogm_update_scans(grid.ctypes.data_as(dp), cfg.ctypes.data_as(dp), W, H, p.ctypes.data_as(dp), p.shape[0],
                                              r.ctypes.data_as(dp), r.shape[1], sc.ANGLE_MIN, sc.ANGLE_INC))
    return ms, grid


def hand_off(sc, g, n=1 << 16):
    f = rr.MonteCarloLocalizer.try_with_initial_state([*sc.truth[0][:3], 1.0], rr.MonteCarloLocalizationConfig(n, n), seed=1)
    out = {}
    out["beam_from_grid_ms"] = timed(lambda: f.set_beam_model_from_grid(g, 0.5))
    out["beam_host_round_trip_ms"] = timed(lambda: f.set_beam_model(rr.obstacles_from_log_odds(g.grid, 0.5), sc.RES))
    out["lfield_from_grid_ms"] = timed(lambda: f.set_likelihood_field_from_grid(g, 0.5))
    out["lfield_host_round_trip_ms"] = timed(lambda: f.set_likelihood_field(rr.obstacles_from_log_odds(g.grid, 0.5), sc.RES))
    f.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--scans", type=int, default=600)
    ap.add_argument("--trace-dir", default="", help="write the profiler traces here (not into the tree)")
    a = ap.parse_args()
    sc = scenarios.ScanScenario(steps=60)
    reps = -(-a.scans // len(sc.scans))
    poses = np.tile(np.array(sc.truth), (reps, 1))[:a.scans]
    scans = np.tile(np.stack(sc.scans), (reps, 1))[:a.scans]
    flusher = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(1024, 1024), seed=1)
    sampler = bench.ClockSampler(0)
    res = {"live_plan_us": [], "traj_plan_ms": [], "traj_big_ms": [], "hand_off": []}
    stats = {}
    mapped = grid_map(sc)
    mapped.update_with_scans(sc.truth, np.stack(sc.scans), sc.ANGLE_MIN, sc.ANGLE_INC)
    for r in range(a.runs):
        order = ["live", "plan", "big", "hand_off"]
        for w in (order if r % 2 == 0 else order[::-1]):
            if w == "live":
                res["live_plan_us"].append(live(sc, flusher))
            elif w == "plan":
                ms, stats["plan"] = traj(sc, poses, scans, flusher)
                res["traj_plan_ms"].append(ms)
            elif w == "big":
                ms, stats["big"] = traj(sc, poses, scans, flusher, cells=8192)
                res["traj_big_ms"].append(ms)
            else:
                res["hand_off"].append(hand_off(sc, mapped))
    out = {"live_plan_us": statistics.median(res["live_plan_us"])}
    for k in ("plan", "big"):
        ms = statistics.median(res[f"traj_{k}_ms"])
        st = stats[k]
        out[f"traj_{k}"] = {"scans": a.scans, "call_ms": ms, "events": st.events, "events_per_s": st.events / (ms * 1e-3),
                            "chunks": st.chunks, "longest_run": st.longest_run, "event_cap": st.event_cap}
    out["hand_off"] = {k: statistics.median(h[k] for h in res["hand_off"]) for k in res["hand_off"][0]}
    clocks = sampler.stop()
    for k, cells in (("plan", 0), ("big", 8192)):
        out[f"traj_{k}"]["kernel_ms"] = profile(sc, poses, scans, cells, a.trace_dir)
    cpu_ms, cpu_grid = cpu_oracle(sc, poses, scans)
    g = grid_map(sc)
    g.update_with_scans(poses, scans, sc.ANGLE_MIN, sc.ANGLE_INC)
    # the glibc oracle and the device differ only where glibc's sin / cos and the contract's differ in the last bit and move a cell
    out["cpu_oracle"] = {"call_ms": cpu_ms, "events_per_s": stats["plan"].events / (cpu_ms * 1e-3),
                         "cells_differing_from_device": int((g.grid.view(np.uint64) != cpu_grid.view(np.uint64)).sum())}
    print(json.dumps({"metric": "occupancy grid mapping", "runs": a.runs, **out, "gpu": bench.gpu_info(0), "clocks": clocks}))


if __name__ == "__main__":
    main()
