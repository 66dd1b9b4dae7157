"""FastSLAM particle counts whose post-kernel weight tile does not fit in shared memory: the post kernel then keeps its tiles in
global memory (fs3_post_kernel<512, true>).  Every run is compared with the CPU oracle bit for bit: the gate, the ancestry of
every resample and the best particle every step, the whole state at the end.

PFGPU_POST_SMEM_CAP=0 forces the global-memory tiles at sizes the oracle checks in seconds (with PFGPU_POST_TILES for the
shape); from about 3.2 M particles on (on an H100; one GPU or sharded: every rank evaluates all weights) the engine takes them
by itself.
Maps stay at 4 or 9 landmarks so that the oracle's side of the big runs stays short.
"""
import ctypes as C
import os

import numpy as np
import pytest

import rust_robotics_b200 as rr
from rust_robotics_b200 import scenarios
from _oracle import OracleFS

pytestmark = pytest.mark.gpu


def _grid3(steps):
    """9 landmarks (3 x 3 grid, 10 m pitch); a 10 m circle (u = (1.0, 0.1)) about the middle: ~7 observations per step"""
    return scenarios.FastSlamScenario(3, (10.0, 0.0, 0.0), (1.0, 0.1), steps)


def _grid2(steps):
    """4 landmarks (2 x 2 grid, 10 m pitch); a 10 m circle about the middle: all 4 observed every step"""
    return scenarios.FastSlamScenario(2, (5.0, -5.0, 0.0), (1.0, 0.1), steps)


def _oracle_fs(oracle, n, m, seed, variant=1, nth=None):
    o = OracleFS(oracle, n, m, seed=seed, variant=variant, nth=n / 1.5 if nth is None else nth)
    oracle.orc_fs_set_threads(o.h, len(os.sched_getaffinity(0)))
    return o


def _exact_cdf_resamples(g):
    out = (C.c_ulonglong * 32)()
    assert g.L.pfgpu_fs_post_trace(g.h, out) == 0
    return int(out[11])


def _run(g, o, sc, steps, variant=1):
    """steps through the scenario on both sides; gate, indices and best particle every step, the whole state at the end"""
    resamples = 0
    for t in range(steps):
        did = g.fastslam_update(sc.control, sc.obs[t]) if variant == 1 else g.fastslam2_update(sc.control, sc.obs[t])
        assert did == bool(o.step(sc.control, sc.obs[t])), f"step {t}: gate"
        if did:
            resamples += 1
            idx, oi = g.last_indices(), o.last_indices()
            assert np.array_equal(idx, oi), f"step {t}: {int((idx != oi).sum())} indices differ, first at {np.flatnonzero(idx != oi)[:4]}"
        assert g.get_best_particle()[0] == o.best(), f"step {t}: best particle"
    _compare(g, o, "end")
    return resamples


def _compare(g, o, what):
    gp, gl = g.state()
    op, ol = o.state()
    assert np.array_equal(gp, op), f"{what}: pose/weight rows {np.flatnonzero((gp != op).any(axis=1))[:5]}"
    assert np.array_equal(gl, ol), f"{what}: landmarks differ for particles {np.flatnonzero((gl != ol).any(axis=(1, 2)))[:5]}"


# ---------------------------------------------------------------- 1. global-memory tiles at small n, forced

@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("tiles,n", [(2, 4096), (3, 5000), (1, 2048), (5, 1 << 14)])
def test_global_tiles_forced_shapes_bit_exact(oracle, monkeypatch, variant, tiles, n):
    """the shapes of test_fastslam_post_kernel_shapes_bit_exact (several values per thread, few tiles; 5000 is not a power of two,
    so its comb is an exact scan) with the weight tiles in global memory"""
    monkeypatch.setenv("PFGPU_POST_SMEM_CAP", "0")
    monkeypatch.setenv("PFGPU_POST_TILES", str(tiles))
    sc = scenarios.FastSlamScenario(6, (25.0, 25.0, 0.0), (1.0, 0.025), 16)
    cls = rr.FastSlam1 if variant == 1 else rr.FastSlam2
    g = cls(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=3)
    k = -(-n // (tiles * 512))
    assert g.post_shape() == (-(-n // (512 * k)), 512, k, "global")
    o = _oracle_fs(oracle, n, sc.m, 3, variant)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    assert _run(g, o, sc, 16, variant) > 0
    assert g.stats().serial_fallbacks == 0


@pytest.mark.parametrize("exact", ["0", "1"])
def test_global_tiles_forced_certified_cdf_bit_exact(oracle, monkeypatch, exact):
    """4 096 particles: the certified CDF (and, with PFGPU_FS_EXACT_CDF=1, the exact S2 and CDF sums) read from the global tile"""
    monkeypatch.setenv("PFGPU_POST_SMEM_CAP", "0")
    monkeypatch.setenv("PFGPU_FS_EXACT_CDF", exact)
    n, steps = 4096, 24
    sc = _grid3(steps)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=11)
    assert g.post_shape()[3] == "global"
    o = _oracle_fs(oracle, n, sc.m, 11)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    resamples = _run(g, o, sc, steps)
    assert resamples > 1 and g.stats().serial_fallbacks == 0
    took_exact = _exact_cdf_resamples(g)
    if exact == "1":
        assert took_exact == resamples
    else:
        assert took_exact < resamples, "the certified CDF was never used"


def test_shared_tiles_by_default(monkeypatch):
    """below the shared-memory limit the engine keeps its tiles on chip; PFGPU_POST_SMEM_CAP only moves them when they exceed it"""
    for cap in (None, str(1 << 20)):
        if cap:
            monkeypatch.setenv("PFGPU_POST_SMEM_CAP", cap)
        g = rr.FastSlam1(1 << 16, 4)
        assert g.post_shape() == (128, 512, 1, "shared")
        g.close()


# ---------------------------------------------------------------- 2. beyond the shared-memory limit, natively

def test_4m_particles_fastslam1_bit_exact(oracle):
    n, steps = 1 << 22, 5
    sc = _grid3(steps)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=5)
    assert g.post_shape()[3] == "global"
    o = _oracle_fs(oracle, n, sc.m, 5)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    assert _run(g, o, sc, steps) >= 2
    assert g.stats().serial_fallbacks == 0


def test_4m_particles_fastslam2_bit_exact(oracle):
    n, steps = 1 << 22, 3
    sc = _grid3(steps)
    g = rr.FastSlam2(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=5)
    o = _oracle_fs(oracle, n, sc.m, 5, variant=2)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    assert _run(g, o, sc, steps, variant=2) >= 1
    assert g.stats().serial_fallbacks == 0


def test_3m_particles_not_power_of_two_bit_exact(oracle):
    """3 500 000 particles (just past what fits in shared memory on an H100): not a power of two, so every resample scans the
    comb exactly"""
    n, steps = 3_500_000, 5
    sc = _grid3(steps)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=5)
    assert g.post_shape()[3] == "global"
    o = _oracle_fs(oracle, n, sc.m, 5)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    assert _run(g, o, sc, steps) >= 1
    assert g.stats().serial_fallbacks == 0


def test_16m_particles_end_to_end_bit_exact(oracle):
    """2^24 particles x 4 landmarks (nth = 0.9 n, so that it resamples within a few steps)"""
    n, steps = 1 << 24, 4
    sc = _grid2(steps)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=0.9 * n), seed=5)
    assert g.post_shape()[3] == "global"
    o = _oracle_fs(oracle, n, sc.m, 5, nth=0.9 * n)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    assert _run(g, o, sc, steps) >= 1
    assert g.stats().serial_fallbacks == 0


# ---------------------------------------------------------------- 3. edge cases at 2^22

def test_4m_particles_edge_cases(oracle):
    n = 1 << 22
    sc = _grid2(3)
    g = rr.FastSlam1(n, sc.m, rr.FsConfig(nth=n / 1.5), seed=11)
    o = _oracle_fs(oracle, n, sc.m, 11)
    g.seed_map(sc.start, sc.landmarks); o.seed_map(sc.start, sc.landmarks)
    z = sc.obs[0]
    assert g.fastslam_update(sc.control, z) == bool(o.step(sc.control, z))
    # all-zero weights: no normalisation, neff = 0 -> resample -> every slot clones particle n-1
    p, l = g.state()
    p[:, 0] = 0.0
    g.set_state(p, l); o.set_state(p, l)
    assert g.fastslam_update(sc.control, sc.obs[1]) is True
    assert o.step(sc.control, sc.obs[1]) == 1
    assert np.all(g.last_indices() == n - 1)
    _compare(g, o, "zero weights")
    # tiny uniform weights: every raw square underflows, so one thread of every CTA walks the 4 M squares for N_eff
    p, l = g.state()
    p[:, 0] = 1e-170
    g.set_state(p, l); o.set_state(p, l)
    assert g.fastslam_update(sc.control, []) is False and o.step(sc.control, []) == 0
    _compare(g, o, "tiny uniform weights")
    assert g.last_neff() == pytest.approx(float(n), rel=1e-9)
    assert g.stats().serial_fallbacks == 0


# ---------------------------------------------------------------- 4. sharded, all ranks in this process

def test_4m_particles_sharded_in_process_bit_exact(oracle):
    """2 ranks on one GPU, 2^22 particles in all: every rank's post kernel evaluates all weights from global-memory tiles"""
    n, steps, world = 1 << 22, 4, 2
    sc = _grid3(steps)
    ranks = rr.FastSlam1.create_sharded_local(n, sc.m, [0] * world, rr.FsConfig(nth=n / 1.5), seed=9)
    assert all(g.post_shape()[3] == "global" for g in ranks)
    o = _oracle_fs(oracle, n, sc.m, 9)
    for g in ranks:
        g.seed_map(sc.start, sc.landmarks)
    o.seed_map(sc.start, sc.landmarks)
    resamples = 0
    for t in range(steps):
        did = rr.FastSlam1.step_all(ranks, sc.control, sc.obs[t])
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
    assert resamples >= 1
    assert all(g.stats().serial_fallbacks == 0 for g in ranks)
