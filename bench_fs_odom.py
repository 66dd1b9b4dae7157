"""bench_fs_odom.py — FastSLAM step time with the velocity and the odometry motion model (DESIGN §3.15), on one GPU.

bench.py's protocol: CUDA events on the engine's stream around every step, L2 flushed before each step, warm-up steps first, the
two motion models alternating in one process, the median step of each reported.  Workloads:
  c3_fs1 / c3_fs2    BASELINE config 3 (65 536 particles x 256 landmarks, c3_scenario's observations), FastSLAM 1.0 / 2.0
  unknown            FastSLAM 2.0 with unknown data association at 65 536 particles x 64 slots
  predict            config 3 without observations: a whole k = 0 step with either model, and the device time of
                     fs3_odom_predict_kernel alone (torch.profiler, CUDA activities, in a separate pass after the timed steps)
The odometry drive follows the scenario's true poses, so both models move the particles by about the same amount.
Prints one JSON line with the card's name, power limit and SM clock.
"""
import argparse
import json
import subprocess

import numpy as np
import torch                      # before libpfgpu.so: torch's CUDA libraries need their own NCCL loaded first
from torch.profiler import ProfilerActivity, profile

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:                                        # noqa: BLE001 - the numbers stand without it
        return {"gpu": f"unknown ({e})"}


def timed_step(g, fn):
    g.flush_l2()
    g.mark(0)
    fn()
    g.mark(1)
    return g.elapsed_ms(0, 1)


def bench(variant, n, m, sc, steps, warmup, unknown=False, no_obs=False):
    cls = rr.FastSlam2 if variant == 2 else rr.FastSlam1
    cfg = rr.FsConfig(nth=n / 1.5)
    g = cls(n, m, cfg, seed=7)
    if unknown:
        g.set_state(np.tile([1.0 / n, *sc.start], (n, 1)), np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, m, 1)))
    else:
        g.seed_map(sc.start, sc.landmarks)
    odo = [list(sc.start)] + [list(p) for p in sc.truth]
    times = {"velocity": [], "odometry": []}
    for t in range(warmup + steps):
        z = [] if no_obs else sc.obs[t % len(sc.obs)]
        zu = [(d, a) for d, a, _ in z]
        a, b = odo[t % len(sc.obs)], odo[t % len(sc.obs) + 1]
        for kind in (("velocity", "odometry") if t % 2 == 0 else ("odometry", "velocity")):
            if kind == "velocity":
                fn = (lambda: g.fastslam2_update_unknown(sc.control, zu, want_flag=False)) if unknown else \
                     (lambda: g.fastslam_update(sc.control, z, want_flag=False))
            else:
                fn = (lambda: g.fastslam2_update_unknown_odometry(a, b, zu, want_flag=False)) if unknown else \
                     (lambda: g.fastslam_update_odometry(a, b, z, want_flag=False))
            ms = timed_step(g, fn)
            if t >= warmup:
                times[kind].append(ms)
    g.sync()
    v, o = float(np.median(times["velocity"])) * 1e3, float(np.median(times["odometry"])) * 1e3
    return {"velocity_us": round(v, 2), "odometry_us": round(o, 2), "ratio": round(o / v, 4)}


def predict_kernel_us(n, sc, steps):
    """mean device time of fs3_odom_predict_kernel over `steps` odometry steps without observations (config 3's shape)"""
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=7)
    g.seed_map(sc.start, sc.landmarks)
    odo = [list(sc.start)] + [list(p) for p in sc.truth]
    for t in range(3):
        g.fastslam_update_odometry(odo[t], odo[t + 1], [], want_flag=False)
    g.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t in range(steps):
            g.fastslam_update_odometry(odo[t % len(sc.obs)], odo[t % len(sc.obs) + 1], [], want_flag=False)
        g.sync()
        torch.cuda.synchronize()
    ts = [e.device_time for e in prof.events() if "fs3_odom_predict_kernel" in e.name]
    assert len(ts) == steps, f"profiled {len(ts)} fs3_odom_predict_kernel launches, expected {steps}"
    return round(float(np.mean(ts)), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    n = 65536
    c3 = scenarios.c3_scenario(steps=args.steps + args.warmup)
    small = scenarios.FastSlamScenario(8, (35.0, 35.0, 0.0), (1.0, 0.025), args.steps + args.warmup, seed=42)
    out = dict(gpu_info())
    out["c3_fs1"] = bench(1, n, c3.m, c3, args.steps, args.warmup)
    out["c3_fs2"] = bench(2, n, c3.m, c3, args.steps, args.warmup)
    out["unknown"] = bench(2, n, 64, small, args.steps, args.warmup, unknown=True)
    out["predict"] = bench(1, n, c3.m, c3, args.steps, args.warmup, no_obs=True)
    out["predict"]["odom_predict_kernel_us"] = predict_kernel_us(n, c3, args.steps)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
