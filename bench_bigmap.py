#!/usr/bin/env python3
"""bench_bigmap.py — how the FastSLAM step time depends on the map size, at a fixed particle count.

    python bench_bigmap.py --steps K --warmup W [--variant 2]          # one JSON line

Measures 2^15 particles x 16 384 landmarks (128 x 128 grid at 10 m pitch, C3's 40 m circle moved to the middle of the grid,
so ~12.7 landmarks are observed per step as in C3; the two map buffers take 51.5 GB and the ancestry rows 4.3 GB, so it
fits one 80 GB H100) and, in the same process, the same particle count on C3's 256-landmark map (key `m256_same_particles`).
Both use bench.py's measurement protocol (`bench.measure`: warm-up, K event-timed steps with L2 flushed before each, K steps
back to back) and report its numbers.  No CPU arm: the oracle deep-copies 786 KB per particle per resample at this map size.
With PFGPU_POST_TRACE=1 the post kernel's phase times of both maps go to stderr.  Writes nothing into the tree.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402

N_PARTICLES = 1 << 15
CONFIGS = {
    "bigmap": dict(name="FastSLAM 1.0 (fs1.rs fastslam_update), 2^15 particles x 16 384 landmarks (128 x 128 grid, C3's circle in the middle)",
                   particles_per_gpu=None, particles_total=N_PARTICLES, scenario="bigmap_scenario", scaling="strong"),
    "bigmap_m256": dict(name="FastSLAM 1.0 (fs1.rs fastslam_update), 2^15 particles x 256 landmarks (C3's map and circle)",
                        particles_per_gpu=None, particles_total=N_PARTICLES, scenario="c3_scenario", scaling="strong"),
}


def summary(r):
    K = r["K"]
    return {"value": r["n_global"] * K / r["t_flushed"], "unit": "particle-steps/s", "steps": K, "ms_per_step": r["t_flushed"] / K * 1e3,
            "value_steady_state_no_flush": r["n_global"] * K / r["t_noflush"], "ekf_launch_ms": r["kernel_ms"],
            "serial_fallbacks": r["serial_fallbacks"],
            "config": bench.workload_config(r["cfg"], r["sc"], 1, r["n_global"], r["obs_timed"], r["resamples"], K)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--variant", type=int, default=1, choices=[1, 2], help="1 = FastSLAM 1.0, 2 = FastSLAM 2.0 on the same maps")
    args = ap.parse_args()
    import rust_robotics_b200 as rr
    from rust_robotics_b200 import dist as rdist
    bench.VARIANT = args.variant
    bench.CONFIGS.update(CONFIGS)
    grp = rdist.TcpGroup(rank=0, world=1)
    K, W = args.steps, max(3, args.warmup)
    big = bench.measure(rr, grp, "bigmap", K, W, 0, 1, 0, False)
    small = bench.measure(rr, grp, "bigmap_m256", K, W, 0, 1, 0, False)
    line = {"metric": "particle-steps/sec", **summary(big), "higher_is_better": True, "dtype": "f64", "data": "synthetic",
            "m256_same_particles": summary(small), "step_time_ratio_16384_over_256": big["t_flushed"] / small["t_flushed"],
            "gpu": bench.gpu_info(0)}
    print(json.dumps(line))
    grp.close()


if __name__ == "__main__":
    main()
