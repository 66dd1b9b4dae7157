#!/usr/bin/env python3
"""bench_path.py — cost of the FastSLAM path history (FastSlam1.enable_history / path / path_estimate; DESIGN §3.6).

    python bench_path.py --steps K --warmup W [--config c3|c4] [--capacity C] [--runs R]          # one JSON line

  - step time with history off and on (capacity C), in R alternating runs of bench.measure's protocol (its scenario and seeded
    map, W warm-up steps, K steps with the L2 flushed before each, an event pair per step); history is enabled right after
    bench.measure seeds the map;
  - fs3_hist_record_kernel's device time from torch.profiler (CUPTI) over a second pass of K steps;
  - once the window is full (C steps after enabling): the path of the best particle and the path moments (path_estimate) for
    L = 100 and L = min(1000, C), as event time on the engine's stream (kernels, copy back, host synchronisation) and host time.
Algorithmic bytes of the record: 28 B read and 28 B written per particle and step, beside the step's 64 + 96 K-bar.  Reports the
card's name, power limit and top SM clock.  Writes nothing into the tree.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402


def record_kernel_us(g, sc, step0, K):
    """mean device time of fs3_hist_record_kernel over K steps (torch.profiler / CUPTI), L2 flushed before each step"""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
    except Exception:              # no usable torch here: kernel times unavailable
        return None
    tot, cnt = 0.0, 0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t in range(K):
            g.flush_l2()
            g.fastslam_update(sc.control, sc.obs[(step0 + t) % len(sc.obs)], want_flag=False)
        g.sync()
    for ev in prof.events():
        if "fs3_hist_record_kernel" in ev.name:
            tot += getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)
            cnt += 1
    return tot / cnt if cnt else None


def timed(g, fn, K):
    fn()                                        # the first call allocates the scratch
    wall = []
    for k in range(K):
        g.flush_l2()
        g.sync()
        g.mark(2 * k)
        t0 = time.perf_counter()
        fn()
        wall.append(time.perf_counter() - t0)
        g.mark(2 * k + 1)
    ev = sorted(g.elapsed_ms(2 * k, 2 * k + 1) * 1e3 for k in range(K))
    return {"event_us_median": ev[K // 2], "host_us_median": sorted(wall)[K // 2] * 1e6}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=100, help="timed steps per run (K)")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--config", default="c3", choices=["c3", "c4"])
    ap.add_argument("--capacity", type=int, default=None, help="history entries (default: 1000 at c3, 64 at c4)")
    ap.add_argument("--runs", type=int, default=3, help="alternating off / on runs")
    ap.add_argument("--queries", type=int, default=20, help="timed calls per query kind")
    args = ap.parse_args()
    try:
        import torch  # noqa: F401  (before libpfgpu.so: torch's CUDA libraries load first)
    except Exception:
        pass
    import rust_robotics_b200 as rr
    from rust_robotics_b200 import dist as rdist, scenarios
    C = args.capacity or (1000 if args.config == "c3" else 64)
    K, W = args.steps, args.warmup
    grp = rdist.TcpGroup()
    # bench.measure seeds the map right after it creates the engine: enable history there when asked
    enable = {"cap": 0}
    seed_map = rr.FastSlam1.seed_map

    def seed_then_enable(self, *a, **kw):
        seed_map(self, *a, **kw)
        if enable["cap"]:
            self.enable_history(enable["cap"])
    rr.FastSlam1.seed_map = seed_then_enable
    runs = {"off": [], "on": []}
    for r in range(args.runs):
        for mode in ("off", "on"):
            enable["cap"] = C if mode == "on" else 0
            res = bench.measure(rr, grp, args.config, K, W, 0, 1, 0, False)
            runs[mode].append({"ms_per_step": res["t_flushed"] / K * 1e3, "launches_per_step": res["launches"] / K,
                               "resamples": res["resamples"]})
    rr.FastSlam1.seed_map = seed_map

    # second pass: the record kernel, then the queries over a full window
    cfg = bench.CONFIGS[args.config]
    n = cfg["particles_total"] or cfg["particles_per_gpu"]
    sc = getattr(scenarios, cfg["scenario"])(steps=max(C, K) + W)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=bench.nth_value(n)), seed=42)
    g.seed_map(sc.start, sc.landmarks)
    for t in range(W):
        g.fastslam_update(sc.control, sc.obs[t], want_flag=False)
    g.enable_history(C)
    rec_us = record_kernel_us(g, sc, W, K)
    for t in range(C):
        g.fastslam_update(sc.control, sc.obs[(W + K + t) % len(sc.obs)], want_flag=False)
    g.sync()
    first, last = g.history_window()
    best = g.get_best_particle()[0]
    queries = {}
    for L in sorted({min(100, C), min(1000, C)}):
        queries[f"path_L{L}"] = timed(g, lambda: g.path(best, L), args.queries)
        queries[f"path_estimate_L{L}"] = timed(g, lambda: g.path_estimate(L), args.queries)
    kbar = sum(len(z) for z in sc.obs[W:W + K]) / K
    med = lambda xs: sorted(xs)[len(xs) // 2]
    off, on = med([x["ms_per_step"] for x in runs["off"]]), med([x["ms_per_step"] for x in runs["on"]])
    line = {"metric": "fastslam path history", "config": args.config, "particles": n, "landmarks": sc.m, "capacity": C,
            "ring_bytes": n * 28 * C, "steps_per_run": K, "warmup": W, "runs": runs,
            "ms_per_step_off_median": off, "ms_per_step_on_median": on, "on_minus_off_us": (on - off) * 1e3,
            "record_kernel_us_mean": rec_us, "record_alg_bytes": n * 56, "step_alg_bytes": n * (64 + 96 * kbar),
            "window": [first, last], "queries": queries, "l2": "flushed before every timed step and call",
            "gpu": bench.gpu_info(0)}
    print(json.dumps(line))
    g.close()


if __name__ == "__main__":
    main()
