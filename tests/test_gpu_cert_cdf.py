"""FastSLAM resample from the certified CDF (DESIGN §1) against the CPU oracle, bit for bit, with and without
PFGPU_FS_EXACT_CDF=1 (every resample runs the exact S2 and CDF sums): power-of-two particle counts take the certified CDF unless
its certificate refuses, other counts always take the exact sums.  FastSLAM 1.0 and 2.0, one GPU and the sharded engine (all
ranks in this process, on one device)."""
import ctypes as C

import numpy as np
import pytest

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
from _oracle import OracleFS

pytestmark = pytest.mark.gpu


def _scenario(steps):
    """C3's map (16 x 16 landmarks at 10 m pitch) and its 40 m circle"""
    return scenarios.FastSlamScenario(16, (75.0, 35.0, 0.0), (1.0, 0.025), steps)


def _exact_cdf_resamples(g):
    out = (C.c_ulonglong * 32)()
    assert g.L.pfgpu_fs_post_trace(g.h, out) == 0
    return int(out[11])


def _check_paths(g, n, resamples, exact):
    took_exact = _exact_cdf_resamples(g)
    pow2 = n & (n - 1) == 0
    if exact or not pow2:
        assert took_exact == resamples
    else:
        assert took_exact < resamples, "the certified CDF was never used"


@pytest.mark.parametrize("exact", ["0", "1"])
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("n,steps", [(1024, 30), (1000, 30), (4096, 24), (32768, 16)])
def test_certified_cdf_trajectory_bit_exact(oracle, monkeypatch, exact, variant, n, steps):
    monkeypatch.setenv("PFGPU_FS_EXACT_CDF", exact)
    sc = _scenario(steps)
    cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2
    g = cls(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=11)
    o = OracleFS(oracle, n, sc.m, seed=11, variant=variant, nth=n / 1.5)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    resamples = 0
    for t in range(steps):
        did = g.fastslam_update(sc.control, sc.obs[t]) if variant == 1 else g.fastslam2_update(sc.control, sc.obs[t])
        assert did == bool(o.step(sc.control, sc.obs[t])), f"step {t}: gate"
        if did:
            resamples += 1
            assert np.array_equal(g.last_indices(), o.last_indices()), f"step {t}: indices"
        assert g.get_best_particle()[0] == o.best(), f"step {t}: best particle"
    gp, gl = g.state()
    op, ol = o.state()
    assert np.array_equal(gp, op) and np.array_equal(gl, ol), "final state differs from the oracle"
    assert resamples > 1
    assert g.stats().serial_fallbacks == 0
    _check_paths(g, n, resamples, exact == "1")


def test_certified_cdf_at_bench_size_bit_exact(oracle):
    """65 536 particles (bench.py's config 3): here the certificate refuses a share of the resamples, whose exact sums then run
    behind the certified pass's grid barrier"""
    n, steps = 65536, 40
    sc = _scenario(steps)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=3)
    o = OracleFS(oracle, n, sc.m, seed=3, nth=n / 1.5)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    resamples = 0
    for t in range(steps):
        did = g.fastslam_update(sc.control, sc.obs[t])
        assert did == bool(o.step(sc.control, sc.obs[t])), f"step {t}: gate"
        if did:
            resamples += 1
            assert np.array_equal(g.last_indices(), o.last_indices()), f"step {t}: indices"
        assert g.get_best_particle()[0] == o.best(), f"step {t}: best particle"
    gp, _ = g.state(False)
    op, _ = o.state()
    assert np.array_equal(gp, op)
    assert resamples > 1 and g.stats().serial_fallbacks == 0
    print(f"65536 particles: {resamples} resamples, {_exact_cdf_resamples(g)} of them on the exact sums")


@pytest.mark.parametrize("exact", ["0", "1"])
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("world,n", [(2, 2048), (4, 4096), (2, 1920), (4, 3840)])
def test_certified_cdf_sharded_in_process_bit_exact(oracle, monkeypatch, exact, variant, world, n):
    monkeypatch.setenv("PFGPU_FS_EXACT_CDF", exact)
    steps = 16
    sc = _scenario(steps)
    cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2
    ranks = cls.create_sharded_local(n, sc.m, [0] * world, rr.FsConfig(nth=n / 1.5), seed=9)
    o = OracleFS(oracle, n, sc.m, seed=9, variant=variant, nth=n / 1.5)
    for g in ranks:
        g.seed_map(sc.start, sc.landmarks)
    o.seed_map(sc.start, sc.landmarks)
    resamples = 0
    for t in range(steps):
        did = cls.step_all(ranks, sc.control, sc.obs[t])
        assert did == bool(o.step(sc.control, sc.obs[t])), f"step {t}: gate"
        if did:
            resamples += 1
            assert np.array_equal(np.concatenate([g.last_indices() for g in ranks]), o.last_indices()), f"step {t}: indices"
        for g in ranks:
            assert g.get_best_particle()[0] == o.best(), f"step {t}: best particle"
    op, ol = o.state()
    for r, g in enumerate(ranks):
        lo, hi = r * g.n_local, (r + 1) * g.n_local
        gp, gl = g.state()
        assert np.array_equal(gp, op[lo:hi]) and np.array_equal(gl, ol[lo:hi]), f"rank {r}: state differs from the oracle"
    assert resamples > 1
    assert all(g.stats().serial_fallbacks == 0 for g in ranks)
    for g in ranks:
        _check_paths(g, n, resamples, exact == "1")
