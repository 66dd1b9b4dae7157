"""pfgpu_pf_stats of the fused PF / MCL step (pf3_post_kernel, one launch after predict + likelihood): its exact sums report
their dirty values and serial walks like the separate kernels' sums do, and the separate kernels (PFGPU_PF_FUSED=0, in a
process of its own: the choice is made when a filter is created) give the same particles."""
import os
import subprocess
import sys

import numpy as np
import pytest

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1 << 16
STEPS = 6


def run(kind):
    """STEPS fused-size steps of a PF (resample every step) or an MCL filter of N particles; returns the filter"""
    if kind == "pf":
        sc = scenarios.PfScenario("c1", steps=STEPS)
        g = rr.ParticleFilterLocalizer.try_with_initial_state(
            (5.0, 5.0, 0.0, 0.0), rr.ParticleFilterConfig(N, 1.0, 0.25, 2.0, np.deg2rad(40.0), 0.1), seed=42)
    else:
        sc = scenarios.PfScenario("c2", steps=STEPS)
        g = rr.MonteCarloLocalizer.try_with_initial_state(
            tuple(sc.init), rr.MonteCarloLocalizationConfig(N, N, 0.05, 2.326, 0.25, 0.05, 0.02, 0.1), seed=5)
    for t in range(STEPS):
        obs = sc.obs[t][:: max(1, sc.obs[t].shape[0] // 24)] if kind == "mcl" else sc.obs[t]
        g.try_step(sc.controls[t], obs)
    return g


def phase_update(g, kind):
    """one update through the phase API: its normalisation is an exact sum of the separate kernels, also with the fused step on"""
    sc = scenarios.PfScenario("c1" if kind == "pf" else "c2", steps=STEPS)
    g.try_update_with_observations(sc.obs[0][:: max(1, sc.obs[0].shape[0] // 24)] if kind == "mcl" else sc.obs[0])
    return g.stats().xsum_dirty_last


@pytest.mark.parametrize("kind", ["pf", "mcl"])
def test_fused_step_reports_its_exact_sums(kind, tmp_path):
    g = run(kind)
    st = g.stats()
    assert st.kernel_launches < 4 * STEPS, "the step did not take the fused tail"
    assert st.resamples == STEPS
    assert st.xsum_dirty_last > 0, "the fused tail's last exact sum reported no dirty values"
    assert st.serial_fallbacks == 0
    parts = g.get_particles()
    dirty_phase = phase_update(g, kind)       # the separate kernels ran the last sum now: their count is reported
    out = tmp_path / "particles.npy"
    script = ("import sys, numpy as np; sys.path[:0] = [sys.argv[1], sys.argv[1] + '/tests']; import test_gpu_pf_fused_stats as t; "
              "g = t.run(sys.argv[2]); assert g.stats().kernel_launches >= 4 * t.STEPS; np.save(sys.argv[3], g.get_particles()); "
              "print('DIRTY', t.phase_update(g, sys.argv[2]))")
    env = dict(os.environ, PFGPU_PF_FUSED="0")
    r = subprocess.run([sys.executable, "-c", script, ROOT, kind, str(out)], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert np.array_equal(parts, np.load(out)), "the fused and the separate kernels' particles differ"
    assert dirty_phase == int(r.stdout.split("DIRTY")[-1]), "after a phase-API update, stats report a stale dirty count"
