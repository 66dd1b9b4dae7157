"""The path history's definition (DESIGN §3.6) on the CPU oracle, before any GPU is involved: the genealogy backtrack through
per-step poses and resample parents, built only from state() and last_indices() after every step, gives bit for bit the list of
past poses each particle would carry if it were cloned with the particle on every resample."""
import numpy as np
import pytest

from rust_robotics_b200 import scenarios
from _oracle import OracleFS
from _assoc_oracle import OracleFS2Assoc
from _path_oracle import Genealogy, VecPaths


def _check(gen, vec, n, what):
    for g in range(n):
        steps, slots, poses = gen.path(g)
        want = vec.paths[g]
        assert [int(s) for s in steps] == [s for s, _ in want], f"{what}: slot {g} steps"
        assert np.array_equal(poses, np.array([p for _, p in want])), f"{what}: slot {g} poses"
        assert slots[-1] == g


def _run(o, n, steps, step_fn, cap=None):
    pw, _ = o.state()
    gen, vec = Genealogy(cap), VecPaths(pw)
    gen.root(0, pw)
    resampled = 0
    for t in range(1, steps + 1):
        did = step_fn(t - 1)
        pw, _ = o.state()
        idx = o.last_indices()
        assert bool(did) == (len(idx) > 0)
        resampled += int(bool(did))
        gen.record(t, pw, idx)
        vec.step(t, pw, idx)
    return gen, vec, resampled


@pytest.mark.parametrize("variant", [1, 2])
def test_backtrack_equals_cloned_lists(oracle, variant):
    n, steps = 64, 16
    sc = scenarios.c3_scenario(steps=steps)
    o = OracleFS(oracle, n, sc.m, seed=3, variant=variant, nth=n / 1.5)
    o.seed_map(sc.start, sc.landmarks)
    gen, vec, resampled = _run(o, n, steps, lambda t: o.step(sc.control, sc.obs[t]))
    assert resampled > 1
    _check(gen, vec, n, f"variant {variant}")
    # a ring smaller than the run holds the tail of every list
    small = Genealogy(5)
    small.entries = gen.entries[-5:]
    for g in range(n):
        steps_, _, poses = small.path(g)
        assert [int(s) for s in steps_] == [s for s, _ in vec.paths[g][-5:]]
        assert np.array_equal(poses, np.array([p for _, p in vec.paths[g][-5:]]))


def test_backtrack_unknown_association():
    n, m, steps = 64, 16, 10
    sc = scenarios.FastSlamScenario(6, (25.0, 5.0, 0.0), (1.0, 0.05), steps, seed=7, max_range=80.0)
    o = OracleFS2Assoc(n, m, seed=5, nth=n / 1.5)
    pw = np.tile([1.0 / n, *sc.start], (n, 1))
    o.set_state(pw, np.tile([0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0], (n, m, 1)))
    gen, vec, resampled = _run(o, n, steps, lambda t: o.step_unknown(sc.control, [(d, a) for d, a, _ in sc.obs[t]]))
    assert resampled > 1
    _check(gen, vec, n, "unknown association")
