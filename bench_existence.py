#!/usr/bin/env python3
"""bench_existence.py — landmark existence counters (DESIGN §3.7) off vs on, on the unknown-association step from a fresh map.

    python bench_existence.py --steps K --warmup W [--configs p16,c3] [--long 1000]      # one JSON line

p16: `particles_scenario`, 2^16 particles x 64 slots; c3: `c3_scenario`, 2^16 x 256.  bench_assoc.py's protocol (`bench.measure`:
L2 flushed before every timed step, one event pair per step, a second pass with events around the association kernel), four runs
alternating off / on, median per setting; removals per step from an untimed run of the same steps.  The long-run block: the
config-3 grid at 2^16 x 64 slots, `--long` steps from a fresh map, off and on: the best particle's initialised slots, landmarks
seen and observations dropped, every 100 steps.  Writes nothing into the tree.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402
import bench_assoc  # noqa: E402

CONFIGS = {
    "p16": (1 << 16, 64, "particles_scenario"),
    "c3": (1 << 16, 256, "c3_scenario"),
}
RANGE = 20.0


def existence_api(rr, slots, on):
    """bench_assoc's unknown-association engine, with counters (range 20 m) when `on`"""
    api = bench_assoc.unknown_api(rr, slots)

    class Tracked(api.FastSlam2):
        def __init__(self, n, m, config=None, **kw):
            super().__init__(n, m, config, **kw)
            if on:
                self.enable_existence(RANGE)
    api.FastSlam1 = api.FastSlam2 = Tracked
    return api


def run(rr, sc, n, m, seed, steps, on, every=0):
    """`steps` untimed steps from a fresh map: removals per step, or (every > 0) the long-run rows"""
    g = rr.FastSlam2(n, m, rr.FsConfig(nth=n / 1.5), seed=seed)
    g.set_state(np.tile([1.0 / n, *sc.start], (n, 1)), np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, m, 1)))
    if on:
        g.enable_existence(RANGE)
    seen, drops, rows, rem = set(), 0, [], []
    for t in range(steps):
        seen |= {l for _, _, l in sc.obs[t]}
        g.fastslam2_update_unknown(sc.control, [(d, a) for d, a, _ in sc.obs[t]], want_flag=False)
        if not every:
            rem.append(g.removed_count())
            continue
        drops += g.assoc_counts()[2]
        if (t + 1) % every == 0:
            lm = g.particle_landmarks(g.get_best_particle()[0])
            rows.append({"step": t + 1, "landmarks_seen": len(seen), "best_initialised_slots": int((lm[:, 2] < 100.0).sum()),
                         "dropped_last_100": int(drops)})
            drops = 0
    g.close()
    return rows if every else rem


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--configs", default="p16,c3")
    ap.add_argument("--long", type=int, default=1000)
    args = ap.parse_args()
    import rust_robotics_b200 as rr
    from rust_robotics_b200 import dist as rdist, scenarios
    grp = rdist.TcpGroup(rank=0, world=1)
    K, W = args.steps, max(3, args.warmup)
    bench.VARIANT = 2
    rows = []
    for key in args.configs.split(","):
        n, slots, scen = CONFIGS[key]
        bench.CONFIGS[key] = dict(name=key, particles_per_gpu=None, particles_total=n, scenario=scen, scaling="strong")
        runs = {False: [], True: []}
        for rep in range(4):                                           # off, on, off, on
            on = rep % 2 == 1
            runs[on].append(bench.measure(existence_api(rr, slots, on), grp, key, K, W, 0, 1, 0, False))
        med = lambda on, f: statistics.median(f(r) for r in runs[on])
        rem = run(rr, getattr(scenarios, scen)(steps=W + 2 * K), n, slots, 42, W + 2 * K, True)[W:]
        rf = med(True, lambda r: r["resamples"] / K)
        row = {"config": key, "particles": n, "slots": slots, "scenario": scen, "range_m": RANGE}
        for on in (False, True):
            tag = "on" if on else "off"
            row[f"us_per_step_{tag}"] = med(on, lambda r: r["t_flushed"] / K * 1e6)
            row[f"assoc_kernel_us_{tag}"] = med(on, lambda r: r["kernel_ms"] * 1e3)
            row[f"runs_us_per_step_{tag}"] = [r["t_flushed"] / K * 1e6 for r in runs[on]]
        row["removals_per_step"] = sum(rem) / len(rem)
        row["resample_fraction_on"] = rf
        row["added_alg_bytes_per_particle_step_max"] = 8 * slots * rf + 32 * slots
        rows.append(row)
    out = {"metric": "us/step", "value": rows[0]["us_per_step_on"], "unit": "us/step", "higher_is_better": False,
           "workload": "FastSLAM 2.0, unknown data association, fresh map, existence counters off vs on (range 20 m)",
           "steps": K, "warmup": W, "l2": "flushed (256 MiB memset + clean read) before every timed step", "configs": rows}
    if args.long:
        sc = scenarios.FastSlamScenario(16, (75.0, 75.0, 0.0), (1.0, 0.025), args.long, seed=42)
        out["long_run"] = {"shape": "config-3 grid, 2^16 particles x 64 slots, fresh map, seed 5",
                           **{k: run(rr, sc, 1 << 16, 64, 5, args.long, on, every=100) for k, on in (("off", False), ("on", True))}}
    out["gpu"] = bench.gpu_info(0)
    print(json.dumps(out))
    grp.close()


if __name__ == "__main__":
    main()
