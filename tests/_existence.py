"""The long-run behaviour of the landmark existence counters (DESIGN §3.7), shared by the CPU oracle test and the GPU test: the
config-3 landmark grid and its 40 m circle, a fresh map of 64 slots, observations without ids.  Test infrastructure only."""
import numpy as np

from rust_robotics_b200 import scenarios

N, M, STEPS, SEED, RANGE = 256, 64, 1000, 5, 20.0
SLACK = 8                     # initialised slots of the best particle beyond the landmarks seen (fixed from the run)


def scenario():
    return scenarios.FastSlamScenario(16, (75.0, 75.0, 0.0), (1.0, 0.025), STEPS, seed=42)


def run(step, best_map, sc, steps=STEPS):
    """step(u, z) -> (dropped, removed) of that step; best_map() -> (m, 6).  Returns per step: landmarks seen so far, initialised
    slots of the best particle (every 100 steps, else -1), drops, removals."""
    seen, out = set(), []
    for t in range(steps):
        seen |= {l for _, _, l in sc.obs[t]}
        dropped, removed = step(sc.control, [(d, a) for d, a, _ in sc.obs[t]])
        slots = int((best_map()[:, 2] < 100.0).sum()) if (t + 1) % 100 == 0 else -1
        out.append((len(seen), slots, dropped, removed))
    return np.array(out, dtype=np.int64)


def check(on, off):
    """with counters: no drops, the best particle's map within SLACK of the landmarks seen; without: the map is full by the end"""
    assert on[:, 2].sum() == 0, on[:, 2].nonzero()
    assert on[:, 3].sum() > 0
    rows = on[on[:, 1] >= 0]
    assert (rows[:, 1] <= rows[:, 0] + SLACK).all(), rows
    assert off[-1, 1] == M and off[-1, 2] > 0 and off[-1, 0] < M
