#!/usr/bin/env python3
"""bench_particles.py — how the FastSLAM step time grows with the particle count, up to 2^24 particles on one GPU.

    python bench_particles.py --steps K --warmup W [--variant 2] [--sizes 16,18,20]       # one JSON line

FastSLAM 1.0 on a 36-landmark map (6 x 6 grid at 10 m pitch); the robot drives a 20 m circle (u = (1.0, 0.05)) about the
middle of the grid and sees ~11 landmarks per step; nth = particles / 1.5.  Sizes 2^16, 2^18, 2^20, 2^21, 2^22, 2^23 and 2^24
(the two map buffers take 2 x 96 x 36 B per particle: 58 GB at 2^24).  Each size uses bench.py's measurement protocol
(`bench.measure`: warm-up, K event-timed steps with L2 flushed before each, K steps back to back) and reports, per size, the
step time, particle-steps/s, the EKF launch time, where the post kernel keeps its weight tiles ("shared" memory, or "global"
memory once a tile no longer fits on chip), the mean number of observations per step and the resample fraction.  With
PFGPU_POST_TRACE=1 the post kernel's phase times of every size go to stderr.  Writes nothing into the tree.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402

SIZES_LOG2 = (16, 18, 20, 21, 22, 23, 24)


def config(log2n):
    return dict(name=f"FastSLAM 1.0 (fs1.rs fastslam_update), 2^{log2n} particles x 36 landmarks (6 x 6 grid, 20 m circle about its middle)",
                particles_per_gpu=None, particles_total=1 << log2n, scenario="particles_scenario", scaling="strong")


def post_shape(rr, n):
    """the post kernel's shape at n particles (it depends on the particle count and the device only, not on the map)"""
    g = rr.FastSlam1(n, 1)
    try:
        tiles, threads, k, where = g.post_shape()
    finally:
        g.close()
    return {"tiles": tiles, "threads": threads, "values_per_thread": k, "weights_in": where}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--variant", type=int, default=1, choices=[1, 2], help="1 = FastSLAM 1.0, 2 = FastSLAM 2.0 on the same map")
    ap.add_argument("--sizes", default=",".join(str(p) for p in SIZES_LOG2), help="comma-separated log2 particle counts")
    args = ap.parse_args()
    import rust_robotics_b200 as rr
    from rust_robotics_b200 import dist as rdist
    bench.VARIANT = args.variant
    grp = rdist.TcpGroup(rank=0, world=1)
    K, W = args.steps, max(3, args.warmup)
    sweep = []
    for p in (int(s) for s in args.sizes.split(",")):
        key = f"particles_2^{p}"
        bench.CONFIGS[key] = config(p)
        shape = post_shape(rr, 1 << p)
        if os.environ.get("PFGPU_POST_TRACE"):
            sys.stderr.write(f"--- 2^{p} particles, post kernel {shape}\n")
        r = bench.measure(rr, grp, key, K, W, 0, 1, 0, False)
        wc = bench.workload_config(r["cfg"], r["sc"], 1, r["n_global"], r["obs_timed"], r["resamples"], K)
        sweep.append({"particles": r["n_global"], "us_per_step": r["t_flushed"] / K * 1e6, "particle_steps_per_s": r["n_global"] * K / r["t_flushed"],
                      "us_per_step_no_flush": r["t_noflush"] / K * 1e6, "ekf_launch_us": r["kernel_ms"] * 1e3, "post_kernel": shape,
                      "mean_obs_per_step": wc["mean_obs_per_step"], "resample_fraction": wc["resample_fraction"],
                      "serial_fallbacks": r["serial_fallbacks"]})
    top = sweep[-1]
    line = {"metric": "particle-steps/sec", "value": top["particle_steps_per_s"], "unit": "particle-steps/s", "particles": top["particles"],
            "higher_is_better": True, "dtype": "f64", "data": "synthetic", "steps": K, "warmup": W,
            "workload": config(0)["name"].replace("2^0 particles", "particle-count sweep") + ("" if args.variant == 1 else " [FastSLAM 2.0 step, fastslam2.rs]"),
            "nth": "particles/1.5", "l2": "flushed (256 MiB memset + clean read) before every timed step",
            "sweep": sweep, "gpu": bench.gpu_info(0)}
    print(json.dumps(line))
    grp.close()


if __name__ == "__main__":
    main()
