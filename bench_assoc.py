#!/usr/bin/env python3
"""bench_assoc.py — the FastSLAM 2.0 step with UNKNOWN data association (pfgpu_fs_step_unknown, DESIGN §3.5) from a fresh map.

    python bench_assoc.py --steps K --warmup W [--configs p16,p20,c3]       # one JSON line

Configurations: `particles_scenario` (36 landmarks on a 6 x 6 grid, 20 m circle about its middle) with 64 landmark slots at 2^16 and
2^20 particles, and the config-3 shape (`c3_scenario`: 16 x 16 grid, 256 slots) at 2^16 particles.  Every particle starts at the
scenario's start pose with an empty map; the observations are the scenario's, without their landmark ids.  Each configuration
uses bench.py's measurement protocol (`bench.measure`: warm-up, K event-timed steps with L2 flushed before each, a second such
pass with events around fs3_assoc_kernel, K steps back to back) and, for contrast, the known-id FastSLAM 2.0 step (pfgpu_fs_step on
a seeded map) on the same scenario and particle count.

Algorithmic bytes per step, two counts: pose and weight read and written (64 B per particle), K + 1 scans over the m slots (the
proposal scan and one per observation), the read and write of each updated landmark (96 B) and, on a step after a resample, the
materialisation of the whole map (read through the rows, written to the other buffer: 96 m B per particle).  A scan reads 48 B of
an initialised slot but only the 8 B of cov00 of an empty one, so `alg_bytes_full` (every slot initialised) bounds the traffic
from above and `alg_bytes_min` (every slot empty) from below; a map fills from empty during the run.  Fractions are of 3.35 TB/s
(H100 SXM data sheet) over the fs3_assoc_kernel time.  Writes nothing into the tree.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402

CONFIGS = {
    "p16": (1 << 16, 64, "particles_scenario"),
    "p20": (1 << 20, 64, "particles_scenario"),
    "c3": (1 << 16, 256, "c3_scenario"),
}


def unknown_api(rr, slots):
    """rr with FastSlam1 / FastSlam2 replaced by an engine whose fastslam_update is the unknown-association step, so that
    bench.measure drives it unchanged: `slots` landmark slots, a fresh map instead of seed_map, observations without ids"""
    class Unknown(rr.FastSlam2):
        def __init__(self, n, m, config=None, **kw):
            super().__init__(n, slots, config, **kw)

        def seed_map(self, pose3, landmarks_xy, sigma=1.0, cov0=10.0):
            n = self.n_local
            self.set_state(np.tile([1.0 / n, *pose3], (n, 1)), np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, self.m, 1)))

        @staticmethod
        def _obs(z):
            return np.ascontiguousarray(np.array([(d, a) for d, a, _ in z], dtype=np.float64).reshape(-1, 2))

        def fastslam_update(self, u, z, want_flag=True, obs_array=None):
            return self.fastslam2_update_unknown(u, obs_array if obs_array is not None else self._obs(z), want_flag=want_flag)

    class Api:
        pass
    api = Api()
    api.__dict__.update({k: getattr(rr, k) for k in dir(rr) if not k.startswith("__")})
    api.FastSlam1 = api.FastSlam2 = Unknown
    return api


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--configs", default="p16,p20,c3")
    args = ap.parse_args()
    import rust_robotics_b200 as rr
    from rust_robotics_b200 import dist as rdist
    grp = rdist.TcpGroup(rank=0, world=1)
    K, W = args.steps, max(3, args.warmup)
    bench.VARIANT = 2
    peak = 3.35e12
    rows = []
    for key in args.configs.split(","):
        n, slots, scen = CONFIGS[key]
        bench.CONFIGS[key] = dict(name=key, particles_per_gpu=None, particles_total=n, scenario=scen, scaling="strong")
        r = bench.measure(unknown_api(rr, slots), grp, key, K, W, 0, 1, 0, False)
        known = bench.measure(rr, grp, key, K, W, 0, 1, 0, False)
        ks = [len(z) for z in r["obs_timed"]]
        kmean = sum(ks) / len(ks)
        rf = r["resamples"] / K
        full = n * (64 + (kmean + 1) * slots * 48 + 96 * kmean + rf * slots * 96)
        low = n * (64 + (kmean + 1) * slots * 8 + 96 * kmean + rf * slots * 96)
        kern_s = r["kernel_ms"] * 1e-3
        rows.append({"config": key, "particles": n, "slots": slots, "scenario": scen, "mean_obs_per_step": round(kmean, 2),
                     "us_per_step": r["t_flushed"] / K * 1e6, "us_per_step_no_flush": r["t_noflush"] / K * 1e6,
                     "assoc_kernel_us": r["kernel_ms"] * 1e3, "alg_bytes_full": full, "alg_bytes_min": low,
                     "bandwidth_fraction_full": full / kern_s / peak if kern_s > 0 else None,
                     "bandwidth_fraction_min": low / kern_s / peak if kern_s > 0 else None,
                     "resample_fraction": round(r["resamples"] / K, 3), "serial_fallbacks": r["serial_fallbacks"],
                     "known_id_us_per_step": known["t_flushed"] / K * 1e6, "known_id_ekf_kernel_us": known["kernel_ms"] * 1e3})
    top = rows[0]
    print(json.dumps({"metric": "us/step", "value": top["us_per_step"], "unit": "us/step", "higher_is_better": False, "dtype": "f64",
                      "data": "synthetic", "steps": K, "warmup": W,
                      "workload": "FastSLAM 2.0 with unknown data association (per-particle Mahalanobis gate 16), fresh map",
                      "nth": "particles/1.5", "l2": "flushed (256 MiB memset + clean read) before every timed step",
                      "configs": rows, "gpu": bench.gpu_info(0)}))
    grp.close()


if __name__ == "__main__":
    main()
