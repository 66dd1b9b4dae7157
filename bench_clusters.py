#!/usr/bin/env python3
"""bench_clusters.py — pose hypotheses (DESIGN §3.10): what one query costs on the GPU, against the route without it.

    python bench_clusters.py [--calls 20] [--warmup 3] [--sizes 16,20] [--workloads track,init,global3,uniform] [--host]

MCL on ScanScenario's floor plan (max_beams 60) at 2^16 and 2^20 particles, the query at its defaults (0.5 m, 24 yaw bins, the 16
heaviest clusters, no per-slot ranks):
  track     after 6 tracking scan steps from the truth (a few bins)
  init      right after init_region over the plan (every bin of the plan occupied: one giant cluster)
  global3   after 3 global scan steps from init_region (multimodal)
  uniform   init_region over the extent of the 8192 x 8192 map at 5 cm, 409.6 m square (nearly every particle its own bin and cluster)
Per workload: the query's time, a host clock around the synchronising call with the L2 flushed before each, the median of `calls`
calls after `warmup`; the kernel time of one query from torch.profiler in a separate pass (CUDA kernels and memsets, summed); the
bins and clusters; and, for contrast, one tracking scan step timed the same way.  --host adds the route callers have without the
query: get_particles() and the numpy restatement of the contract (tests/_cluster_oracle.py) on the host.  The card's name, power
limit and SM clock are on the same JSON line.  Writes nothing into the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch  # noqa: F401  (torch.profiler; loaded before libpfgpu.so so that torch's NCCL is the one resolved)

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402
import rust_robotics_b200 as rr  # noqa: E402
from rust_robotics_b200 import scenarios  # noqa: E402

UNIFORM = (-204.8, 204.8, -204.8, 204.8)


def make(key, sc, n):
    cfg = rr.MonteCarloLocalizationConfig(n, n, 0.05, 2.326, 0.25, 0.2, 0.1, 0.1)
    g = rr.MonteCarloLocalizer.try_with_initial_state([*sc.truth[0][:3], 1.0], cfg, seed=42)
    g.set_likelihood_field(sc.obstacles, sc.RES, max_beams=60)
    if key == "track":
        for t in range(6):
            g.try_step_scan(sc.controls[t], *sc.scan_args(t), want_estimate=False)
    elif key in ("init", "global3"):
        g.init_region(sc.REGION)
        for t in range(3 if key == "global3" else 0):
            g.try_step_scan(sc.controls[t], *sc.scan_args(t), want_estimate=False)
    else:
        g.init_region(UNIFORM)
    g.sync()
    return g


def timed(g, f, calls, warmup):
    for _ in range(warmup):
        f()
    ts = []
    for _ in range(calls):
        g.flush_l2()
        g.sync()
        t0 = time.perf_counter()
        f()
        ts.append((time.perf_counter() - t0) * 1e6)
    return statistics.median(ts)


def kernel_us(g, reps=5):
    """device time of the CUDA kernels and memsets of one query (torch.profiler, a pass of its own)"""
    from torch.profiler import ProfilerActivity, profile
    g.hypotheses()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            g.hypotheses()
    tot = 0.0
    for e in prof.key_averages():
        tot += getattr(e, "self_device_time_total", getattr(e, "self_cuda_time_total", 0.0))
    return tot / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="16,20")
    ap.add_argument("--workloads", default="track,init,global3,uniform")
    ap.add_argument("--host", action="store_true")
    a = ap.parse_args()
    sc = scenarios.ScanScenario(steps=60)
    sampler = bench.ClockSampler(0)
    out = {}
    for lg in [int(s) for s in a.sizes.split(",") if s]:
        n = 1 << lg
        g = make("track", sc, n)
        t = [6]

        def scan_step():
            g.try_step_scan(sc.controls[t[0] % 60], *sc.scan_args(t[0] % 60), want_estimate=False)
            g.sync()
            t[0] += 1
        out[f"scan_step_2^{lg}"] = {"particles": n, "us": timed(g, scan_step, a.calls, a.warmup)}
        g.close()
        for key in [k for k in a.workloads.split(",") if k]:
            g = make(key, sc, n)
            hs, total = g.hypotheses()
            res = {"particles": n, "clusters": total, "bins": int(sum(h.bins for h in g.hypotheses(total)[0])),
                   "top_mass": hs[0].weight if hs else None, "query_us": timed(g, g.hypotheses, a.calls, a.warmup)}
            res["query_kernel_us"] = kernel_us(g)
            if a.host:
                sys.path.insert(0, os.path.join(ROOT, "tests"))
                import _cluster_oracle
                res["get_particles_us"] = timed(g, g.get_particles, 3, 1)
                p = g.get_particles()
                t0 = time.perf_counter()
                _cluster_oracle.hypotheses(p)
                res["host_clustering_us"] = (time.perf_counter() - t0) * 1e6
            out[f"{key}_2^{lg}"] = res
            g.close()
    print(json.dumps({"metric": "pose hypotheses query", "calls": a.calls, "warmup": a.warmup, "workloads": out, "gpu": bench.gpu_info(0),
                      "clocks": sampler.stop()}))


if __name__ == "__main__":
    main()
