#!/usr/bin/env python3
"""bench_estimate.py — cost of the FastSLAM estimate (FastSlam1.estimate: pfgpu_fs_moments + pfgpu_fs_estimate_merge).

    python bench_estimate.py --steps K --warmup W [--config c3|c4] [--variant 2]          # one JSON line

Builds bench.py's state (its scenario, seeded map, W warm-up steps), then times, with the L2 flushed before each call:
  - K map estimates (every landmark, the default cov00 < 100 filter) and K pose-only estimates, each as
      * event time on the engine's stream (pfgpu_fs_mark / pfgpu_fs_elapsed_ms) from just before the call to just after it
        returns: the kernels, the copy of the moments to the host and the host's synchronisation;
      * kernel time of the fs3_est_* kernels from torch.profiler (CUPTI) over a separate pass of K calls, which the fraction
        of HBM bandwidth is computed from;
  - once (config 3 only): state() plus the same estimate in numpy, the route a caller had before.
Algorithmic bytes: n * 32 (weight and pose) for the pose, plus n * m * 48 (six f64 per landmark copy) for the map; the 4-byte
ancestry-row entries read for landmarks that sit behind a row are reported on their own.  Writes nothing into the tree.
"""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402


def numpy_estimate(pw, lm, c, cov00_max=100.0):
    """the estimate's definition (DESIGN §3.4) in numpy, for the contrast run"""
    import numpy as np
    w = pw[:, 0]
    W = w.sum()
    wrap = lambda a: np.where(np.abs(a) <= math.pi, a, a - 2.0 * math.pi * np.rint(a / (2.0 * math.pi)))
    d = np.stack([pw[:, 1] - c[0], pw[:, 2] - c[1], wrap(pw[:, 3] - c[2])], axis=1)
    a = (w[:, None] * d).sum(axis=0) / W
    e = d - a
    pose_cov = np.einsum("i,ij,ik->jk", w, e, e) / W
    sel = lm[:, :, 2] < cov00_max
    ws = np.where(sel, w[:, None], 0.0)
    sw = ws.sum(axis=0)
    with np.errstate(invalid="ignore", divide="ignore"):
        mx, my = (ws * lm[:, :, 0]).sum(axis=0) / sw, (ws * lm[:, :, 1]).sum(axis=0) / sw
        dx, dy = lm[:, :, 0] - mx, lm[:, :, 1] - my
        cov = np.stack([(ws * (lm[:, :, 2] + dx * dx)).sum(axis=0), (ws * (lm[:, :, 3] + dx * dy)).sum(axis=0),
                        (ws * (lm[:, :, 4] + dx * dy)).sum(axis=0), (ws * (lm[:, :, 5] + dy * dy)).sum(axis=0)], axis=1) / sw[:, None]
    return c + a, pose_cov, sw / W, np.stack([mx, my], axis=1), cov


def kernel_us(g, K, landmarks):
    """mean device time per call of the fs3_est_* kernels (torch.profiler / CUPTI), L2 flushed before each call"""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
    except Exception:              # no usable torch here: kernel times unavailable, the event times still stand
        return None
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(K):
            g.flush_l2()
            g.moments(100.0, landmarks)
    tot = 0.0
    for ev in prof.events():
        if ev.name.startswith("fs3_est_") or "fs3_est_" in ev.name:
            tot += getattr(ev, "device_time", None) or getattr(ev, "cuda_time", 0.0)
    return tot / K


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50, help="timed estimate calls of each kind")
    ap.add_argument("--warmup", type=int, default=20, help="FastSLAM steps before the estimate (bench.py's warm-up)")
    ap.add_argument("--config", default="c3", choices=["c3", "c4"])
    ap.add_argument("--variant", type=int, default=1, choices=[1, 2])
    args = ap.parse_args()
    try:
        import torch  # noqa: F401  (before libpfgpu.so: torch's CUDA libraries load first)
    except Exception:
        pass
    import numpy as np
    import rust_robotics_b200 as rr
    from rust_robotics_b200 import scenarios
    bench.VARIANT = args.variant
    cfg = bench.CONFIGS[args.config]
    n = cfg["particles_total"] or cfg["particles_per_gpu"]
    K, W = args.steps, max(3, args.warmup)
    sc = getattr(scenarios, cfg["scenario"])(steps=W)
    g = (rr.FastSlam2 if args.variant == 2 else rr.FastSlam1)(n, sc.m, rr.FsConfig(nth=bench.nth_value(n)), seed=42)
    g.seed_map(sc.start, sc.landmarks)
    behind_row = np.zeros(sc.m, dtype=bool)     # the lazy clone: a resample puts every landmark not behind a row behind one
    for t in range(W):
        did = g.fastslam_update(sc.control, sc.obs[t])
        for _, _, l in sc.obs[t]:
            behind_row[l] = False
        if did:
            behind_row[:] = True
    g.sync()
    peak_gbs, peak_src = bench.load_peaks()

    def timed(landmarks):
        g.moments(100.0, landmarks)             # the first call allocates the scratch
        ev, wall = [], []
        for k in range(K):
            g.flush_l2()
            g.sync()
            g.mark(2 * k)
            t0 = time.perf_counter()
            g.moments(100.0, landmarks)
            wall.append(time.perf_counter() - t0)
            g.mark(2 * k + 1)
        ev = [g.elapsed_ms(2 * k, 2 * k + 1) * 1e3 for k in range(K)]
        return sorted(ev)[K // 2], sorted(wall)[K // 2] * 1e6

    res = {}
    for name, landmarks in (("map", True), ("pose_only", False)):
        ev_us, wall_us = timed(landmarks)
        k_us = kernel_us(g, K, landmarks)
        alg = n * 32 + (n * sc.m * 48 if landmarks else 0)
        res[name] = {"event_us_median": ev_us, "host_us_median": wall_us, "kernel_us_mean": k_us, "alg_bytes": alg,
                     "row_bytes": int(n * 4 * behind_row.sum()) if landmarks else 0,
                     "hbm_fraction": (alg / (k_us * 1e-6)) / (peak_gbs * 1e9) if k_us else None}
    contrast = None
    if args.config == "c3":
        t0 = time.perf_counter()
        pw, lm = g.state()
        t1 = time.perf_counter()
        numpy_estimate(pw, lm, pw[-1, 1:4])
        t2 = time.perf_counter()
        contrast = {"state_ms": (t1 - t0) * 1e3, "numpy_estimate_ms": (t2 - t1) * 1e3, "download_bytes": int(pw.nbytes + lm.nbytes)}
    line = {"metric": "fastslam estimate", "config": args.config, "variant": args.variant, "particles": n, "landmarks": sc.m,
            "landmarks_behind_row": int(behind_row.sum()), "calls": K, "l2": "flushed before every call", **res,
            "state_plus_numpy": contrast, "peak_gbs": peak_gbs, "peak_source": peak_src, "gpu": bench.gpu_info(0)}
    print(json.dumps(line))
    g.close()


if __name__ == "__main__":
    main()
