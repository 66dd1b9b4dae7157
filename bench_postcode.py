#!/usr/bin/env python3
"""bench_postcode.py — what the FastSLAM post kernel pays for fetching its instructions from HBM, at config 3.

    PFGPU_POST_TRACE=1 python bench_postcode.py --steps K --warmup W [--runs R]        # one JSON line

bench.py flushes the L2 before every step, so the post kernel's ~126 KB of code comes from HBM on every step.  This script
separates that cost from the rest with bench.py's own experiment switches, through `bench.measure` (warm-up, K event-timed
steps with or without the flush, K more with an event pair around the EKF launch, K back to back):

  * no observations (BENCH_EMPTY_OBS=1): the EKF launch moves ~1.5 MB, so without the flush (BENCH_FLUSH_MODE=none) the post
    kernel's code stays in L2 from one step to the next.  Its weights are in L2 either way (the EKF launch has just written
    them), so the gap between the flushed ("cold") and unflushed ("warm") runs is close to the cost of fetching code from HBM
    rather than from L2 (plus the EKF launch's own code and its 1.5 MB, which the trace's EKF slot shows);
  * the same pair resampling every step (bench.py's --nth every), which runs the certified CDF, the search and the clone; the
    clone's pose and row reads are warm too in the unflushed run, so that gap is an upper bound;
  * normal config 3 once, for the phase budget of the build.

Cold and warm runs alternate, R of each.  Step times are the flushed-pass step times `value` is quoted on.  The trace
(PFGPU_POST_TRACE=1, per launch, CTA 0) accumulates over every launch of an engine: in a cold run 2K of its W + 3K steps
are flushed, so the JSON also gives the post launch slot of a flushed step alone, solved from the cold and warm averages.
The trace tables go to stderr.  Writes nothing into the tree.
"""
import argparse
import io
import json
import os
import re
import statistics
import sys

os.environ.setdefault("PFGPU_POST_TRACE", "1")     # read when an engine is created

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True     # importing bench.py must not leave a cache in the tree

import bench  # noqa: E402

# trace fields bench.measure prints, by the label it prints them under
FIELDS = {"load_offsets": r"load\+offsets=([\d.]+)", "s_sum": r"S sum=([\d.]+)", "normalise_gate": r"normalise\+gate=([\d.]+)",
          "cdf_scan": r"CDF scan=([\d.]+)", "comb_barrier": r"comb\+barrier=([\d.]+)", "search_clone": r"search\+clone=([\d.]+)",
          "ekf_launch": r"EKF launch=([\d.]+)", "post_launch": r"post launch=([\d.]+)", "idle_between": r"idle between=([\d.]+)"}


class Tee(io.TextIOBase):
    """stderr that also keeps what was written"""
    def __init__(self, real):
        self.real, self.buf = real, []

    def write(self, s):
        self.real.write(s)
        self.buf.append(s)
        return len(s)

    def flush(self):
        self.real.flush()


def run(rr, grp, K, W, empty, flush, nth):
    os.environ.pop("BENCH_EMPTY_OBS", None)
    if empty:
        os.environ["BENCH_EMPTY_OBS"] = "1"
    os.environ["BENCH_FLUSH_MODE"] = "flush" if flush else "none"
    bench.NTH_MODE = nth
    tee = Tee(sys.stderr)
    sys.stderr = tee
    try:
        r = bench.measure(rr, grp, "c3", K, W, 0, 1, 0, False)
    finally:
        sys.stderr = tee.real
    text = "".join(tee.buf)
    trace = {k: float(m.group(1)) for k, p in FIELDS.items() if (m := re.search(p, text))}
    return {"us_per_step": r["t_flushed"] / K * 1e6, "resamples": r["resamples"], "trace": trace}


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "runs": [round(x, 3) for x in xs]}


def pair(rr, grp, K, W, R, nth):
    cold, warm = [], []
    for i in range(R):
        sys.stderr.write(f"--- {nth}: run {i + 1}/{R}, flushed (cold code)\n")
        cold.append(run(rr, grp, K, W, True, True, nth))
        sys.stderr.write(f"--- {nth}: run {i + 1}/{R}, not flushed (warm code)\n")
        warm.append(run(rr, grp, K, W, True, False, nth))
    c = [x["us_per_step"] for x in cold]
    w = [x["us_per_step"] for x in warm]
    out = {"cold_us_per_step": spread(c), "warm_us_per_step": spread(w), "gap_us": statistics.median(c) - statistics.median(w)}
    pc = [x["trace"].get("post_launch") for x in cold]
    pw = [x["trace"].get("post_launch") for x in warm]
    if None not in pc and None not in pw:
        # cold engine's average = (2K flushed + (W + K) unflushed) / (W + 3K); the unflushed share is taken from the warm runs
        pcs, pws = statistics.median(pc), statistics.median(pw)
        flushed_only = (pcs * (W + 3 * K) - pws * (W + K)) / (2 * K)
        out.update(post_launch_cold_trace_us=spread(pc), post_launch_warm_trace_us=spread(pw),
                   post_launch_flushed_step_us=flushed_only, post_launch_gap_us=flushed_only - pws)
    out["trace_cold_last"], out["trace_warm_last"] = cold[-1]["trace"], warm[-1]["trace"]
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3, help="cold and warm runs of each pair (alternated)")
    args = ap.parse_args()
    import rust_robotics_b200 as rr
    from rust_robotics_b200 import dist as rdist
    grp = rdist.TcpGroup(rank=0, world=1)
    K, W = args.steps, max(3, args.warmup)
    line = {"metric": "post kernel code-fetch gap (us per step)", "steps": K, "warmup": W, "gpu": bench.gpu_info(0),
            "no_resample": pair(rr, grp, K, W, args.runs, "default"),
            "resample_every_step": pair(rr, grp, K, W, args.runs, "every")}
    sys.stderr.write("--- config 3 as bench.py runs it\n")
    line["config3"] = run(rr, grp, K, W, False, True, "default")
    line["gpu_after"] = bench.gpu_info(0)
    print(json.dumps(line))
    grp.close()


if __name__ == "__main__":
    main()
