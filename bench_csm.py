#!/usr/bin/env python3
"""bench_csm.py — correlative scan matching on the device (DESIGN §3.13): what scoring a search window costs, against the sequential
reference rule on one host thread.

    python bench_csm.py [--runs 5] [--trace-dir DIR]

Every workload matches ScanScenario's 360-beam scans (the finite beams, about 360 points) against the table built from a device
OccupancyGridMap of the 800 x 600 floor plan at 5 cm (set_reference_from_grid):
  default      the reference's defaults (+-1 m at 0.1 m, +-0.2 rad at 0.02 rad: 9 261 candidates), one scan per call from a noisy
               odometry pose; median call time over the 60 scans, host clock around the synchronising call, L2 flushed before each
  batch60      all 60 scans in one call (Q = 60) with the same config and poses, against 60 single calls
  reloc        +-2 m at 2.5 cm and +-pi at 0.5 degrees (161 x 161 x 721 = 1.87e7 candidates), one scan
  table        the table build at 5 cm: from host points (the plan's obstacle cell centres) and from the device grid
  cpu_oracle   tests/host/csm_oracle.c built with glibc libm into a temporary directory, one host thread: `default` on one scan, and
               `reloc` on a SUBSET of 9 yaws (+-2 degrees at 0.5 degrees), labelled as such
A lookup is one candidate-point evaluation.  Gathered bytes are 4 + 4 index bytes and 8 table bytes per lookup.  Kernel times come from
torch.profiler in a pass of its own.  Runs alternate their order; medians are reported.  The card's name, power limit and SM clock are
on the same JSON line.  Writes nothing into the tree.
"""
import argparse
import ctypes as C
import json
import math
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

DEFAULT = rr.CorrelativeScanMatcherConfig()
RELOC = rr.CorrelativeScanMatcherConfig(2.0, math.pi, 0.025, math.pi / 360.0, 0.05)
RELOC_SUBSET = rr.CorrelativeScanMatcherConfig(2.0, 4.0 * math.pi / 360.0, 0.025, math.pi / 360.0, 0.05)


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def offsets(rng, step):
    n = int(math.floor(abs(rng / step) + 0.5)) * (1 if rng >= 0 else -1)
    return 2 * n + 1 if n >= 0 else 0


def candidates(cfg):
    return offsets(cfg.linear_search_range, cfg.linear_step) ** 2 * offsets(cfg.angular_search_range, cfg.angular_step)


def scan_points(sc, t):
    r = sc.scans[t]
    a = sc.ANGLE_MIN + np.arange(r.size) * sc.ANGLE_INC
    ok = np.isfinite(r) & (r > 0.0)
    return r[ok] * np.cos(a[ok]), r[ok] * np.sin(a[ok])


def noisy_poses(sc, seed=3):
    rng = np.random.default_rng(seed)
    return np.array(sc.truth) + rng.normal(0.0, 1.0, (len(sc.truth), 3)) * [0.3, 0.3, 0.08]


def plan_grid(sc):
    W, H = sc.obstacles.shape
    g = rr.OccupancyGridMap(rr.OccupancyGridConfig(resolution=sc.RES, width=W, height=H))
    g.set_grid(np.where(sc.obstacles, 2.0, -2.0))
    return g


def rate(ms, lookups):
    return {"call_ms": ms, "lookups": lookups, "lookups_per_s": lookups / (ms * 1e-3), "gathered_bytes": 16 * lookups,
            "gathered_bytes_per_s": 16 * lookups / (ms * 1e-3)}


def run_default(m, sc, pts, poses, flusher):
    for t in range(3):
        m.match(*pts[t], poses[t], DEFAULT)
    ms = []
    for t in range(len(pts)):
        flusher.flush_l2()
        flusher.sync()
        ms.append(timed(lambda: m.match(*pts[t], poses[t], DEFAULT)))
    return statistics.median(ms)


def run_batch(m, pts, poses, flusher):
    qx, qy = [p[0] for p in pts], [p[1] for p in pts]
    m.match(qx, qy, poses, DEFAULT)
    flusher.flush_l2()
    flusher.sync()
    one = timed(lambda: m.match(qx, qy, poses, DEFAULT))
    flusher.flush_l2()
    flusher.sync()
    each = timed(lambda: [m.match(*pts[t], poses[t], DEFAULT) for t in range(len(pts))])
    return one, each


def run_reloc(m, pts, pose, flusher):
    m.match(*pts, pose, RELOC)
    flusher.flush_l2()
    flusher.sync()
    return timed(lambda: m.match(*pts, pose, RELOC))


def run_table(sc, rx, ry, g):
    a = rr.CorrelativeScanMatcher()
    a.set_reference(rx, ry)
    a.table_info(0.05)                          # warm-up: the table's memory is allocated, the builds below only fill it
    a.set_reference_from_grid(g, 0.5)           # and the grid hand-off's mask, index and CUB buffers
    a.table_info(0.05)
    host = timed(lambda: (a.set_reference(rx, ry), a.table_info(0.05)))
    grid = timed(lambda: (a.set_reference_from_grid(g, 0.5), a.table_info(0.05)))
    a.close()
    return host, grid


def profile(m, pts, poses, outdir):
    """per-kernel device time of one default batch and one relocalisation call (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile as prof
    qx, qy = [p[0] for p in pts], [p[1] for p in pts]
    out = {}
    for name, fn in (("batch60", lambda: m.match(qx, qy, poses, DEFAULT)), ("reloc", lambda: m.match(*pts[30], poses[30], RELOC))):
        fn()
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            fn()
            torch.cuda.synchronize()
        split = {}
        for e in p.key_averages():
            kind = next((k for k in ("trig", "cells", "score", "reduce", "best_init") if f"pf_csm_{k}_kernel" in e.key), None)
            if kind is None:
                kind = "copy" if "Memcpy" in e.key or "Memset" in e.key else "other"
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            split[kind] = split.get(kind, 0.0) + t / 1e3
        out[name] = {k: round(v, 4) for k, v in sorted(split.items())}
        if outdir:
            os.makedirs(outdir, exist_ok=True)
            p.export_chrome_trace(os.path.join(outdir, f"csm_{name}.pt.trace.json"))
    return out


def cpu_oracle(rx, ry, pts, pose0, pose_r):
    tmp = tempfile.mkdtemp()
    lib = os.path.join(tmp, "libcsm_oracle_libm.so")
    subprocess.run(["gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-DPF_ORACLE_LIBM", "-shared", "-o",
                    lib, os.path.join(ROOT, "tests", "host", "csm_oracle.c"), "-lm"], check=True)
    L = C.CDLL(lib)
    dp = C.POINTER(C.c_double)
    L.orc_csm_match.restype = None
    L.orc_csm_match.argtypes = [dp, dp, C.c_size_t, dp, dp, C.c_size_t, dp, dp, dp, C.POINTER(C.c_uint64)]
    rx, ry = np.ascontiguousarray(rx), np.ascontiguousarray(ry)

    def one(q, pose, cfg):
        qx, qy = np.ascontiguousarray(q[0]), np.ascontiguousarray(q[1])
        c = np.array([cfg.linear_search_range, cfg.angular_search_range, cfg.linear_step, cfg.angular_step, cfg.grid_resolution])
        p, out, n = np.ascontiguousarray(pose, dtype=np.float64), np.zeros(5), C.c_uint64()
        ms = timed(lambda: L.orc_csm_match(rx.ctypes.data_as(dp), ry.ctypes.data_as(dp), rx.size, qx.ctypes.data_as(dp),
                                           qy.ctypes.data_as(dp), qx.size, p.ctypes.data_as(dp), c.ctypes.data_as(dp), out.ctypes.data_as(dp),
                                           C.byref(n)))
        return ms, int(n.value) * qx.size
    d_ms, d_look = one(pts[0], pose0, DEFAULT)
    r_ms, r_look = one(pts[30], pose_r, RELOC_SUBSET)
    return {"default": {"call_ms": d_ms, "lookups_per_s": d_look / (d_ms * 1e-3)},
            "reloc_subset_9_yaws": {"call_ms": r_ms, "lookups": r_look, "lookups_per_s": r_look / (r_ms * 1e-3)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--trace-dir", default="", help="write the profiler traces here (not into the tree)")
    a = ap.parse_args()
    sc = scenarios.ScanScenario(steps=60)
    pts = [scan_points(sc, t) for t in range(len(sc.scans))]
    poses = noisy_poses(sc)
    npts = [p[0].size for p in pts]
    g = plan_grid(sc)
    m = rr.CorrelativeScanMatcher()
    m.set_reference_from_grid(g, 0.5)
    W, H = sc.obstacles.shape
    ix, iy = np.nonzero(sc.obstacles)
    rx, ry = ((ix + 0.5) - W / 2.0) * sc.RES, ((iy + 0.5) - H / 2.0) * sc.RES
    flusher = rr.MonteCarloLocalizer(rr.MonteCarloLocalizationConfig(1024, 1024), seed=1)
    sampler = bench.ClockSampler(0)
    res = {"default": [], "batch_one": [], "batch_each": [], "reloc": [], "table_host": [], "table_grid": []}
    for r in range(a.runs):
        order = ["default", "batch", "reloc", "table"]
        for w in (order if r % 2 == 0 else order[::-1]):
            if w == "default":
                res["default"].append(run_default(m, sc, pts, poses, flusher))
            elif w == "batch":
                one, each = run_batch(m, pts, poses, flusher)
                res["batch_one"].append(one)
                res["batch_each"].append(each)
            elif w == "reloc":
                res["reloc"].append(run_reloc(m, pts[30], poses[30], flusher))
            else:
                host, grid = run_table(sc, rx, ry, g)
                res["table_host"].append(host)
                res["table_grid"].append(grid)
    med = {k: statistics.median(v) for k, v in res.items()}
    cd, cr = candidates(DEFAULT), candidates(RELOC)
    out = {"reference_points": int(rx.size), "query_points": {"min": min(npts), "max": max(npts), "mean": float(np.mean(npts))},
           "default": dict(rate(med["default"], cd * int(np.median(npts))), candidates=cd),
           "batch60_one_call": dict(rate(med["batch_one"], cd * sum(npts)), candidates=cd * len(pts)),
           "batch60_60_calls": dict(rate(med["batch_each"], cd * sum(npts)), candidates=cd * len(pts)),
           "reloc": dict(rate(med["reloc"], cr * npts[30]), candidates=cr),
           "table_ms": {"from_host_points": med["table_host"], "from_grid": med["table_grid"]}}
    clocks = sampler.stop()
    out["kernel_ms"] = profile(m, pts, poses, a.trace_dir)
    out["cpu_oracle_glibc_one_thread"] = cpu_oracle(rx, ry, pts, poses[0], poses[30])
    print(json.dumps({"metric": "correlative scan matching", "runs": a.runs, **out, "gpu": bench.gpu_info(0), "clocks": clocks}))


if __name__ == "__main__":
    main()
